/*
 * dvo_oracle.cpp -- CPU ORACLE (test infrastructure only; see dvo_oracle.h header).
 * PARITY UNPINNED against the reference (no reference tests / goldens exist, reference not
 * buildable here).  Restatement of tum-vision/dvo_slam dvo_core; citations are relative to
 * the root of a dvo_slam checkout at d25b65bf.
 *
 * Build: see oracle/Makefile (-O2 -msse3 -mfma -ffp-contract=off -frounding-math; NO -ffast-math).
 *  -ffp-contract=off : the reference's mul/add order is kept unfused (its 2012 targets had no
 *                      FMA); fused arithmetic appears only where written as std::fmaf (MIRROR).
 *  -frounding-math   : the residual loop runs under MXCSR round-toward-zero like the reference.
 */
#include "dvo_oracle.h"

#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <vector>

#include <xmmintrin.h>
#include <pmmintrin.h>

namespace {

const float kNaNf = std::numeric_limits<float>::quiet_NaN();
const double kNaN = std::numeric_limits<double>::quiet_NaN();

// ------------------------------------------------------------------------------------------
// image model
// ------------------------------------------------------------------------------------------
struct Level {
  int w = 0, h = 0;
  float fx = 0, fy = 0, ox = 0, oy = 0;
  std::vector<float> ch[6];  // I, Z, Ix, Iy, Zx, Zy
};

}  // namespace

struct orc_pyramid {
  std::vector<Level> levels;
};

namespace {

// rgbd_image.cpp:38-55 pyrDownMeanSmooth<float>: ((a+b)+c)+d then /4.0f
void pyr_down_mean(const std::vector<float>& in, int w, int h, std::vector<float>& out) {
  int ow = w / 2, oh = h / 2;
  out.resize(size_t(ow) * oh);
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) {
      int x0 = 2 * x, x1 = x0 + 1, y0 = 2 * y, y1 = y0 + 1;
      float s = in[size_t(y0) * w + x0] + in[size_t(y0) * w + x1];
      s = s + in[size_t(y1) * w + x0];
      s = s + in[size_t(y1) * w + x1];
      out[size_t(y) * ow + x] = s / 4.0f;
    }
}

// rgbd_image.cpp:127-139 pyrDownSubsample<float>
void pyr_down_subsample(const std::vector<float>& in, int w, int h, std::vector<float>& out) {
  int ow = w / 2, oh = h / 2;
  out.resize(size_t(ow) * oh);
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) out[size_t(y) * ow + x] = in[size_t(2 * y) * w + 2 * x];
}

// rgbd_image.cpp:419-433 calculateDerivativeX / 458-472 calculateDerivativeY and
// rgbd_image_sse.cpp:241-284 (same formula): (img[next]-img[prev])*0.5f, indices clamped.
void derivative_x(const std::vector<float>& in, int w, int h, std::vector<float>& out) {
  out.resize(size_t(w) * h);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      int prev = x - 1 < 0 ? 0 : x - 1;
      int next = x + 1 > w - 1 ? w - 1 : x + 1;
      out[size_t(y) * w + x] = (in[size_t(y) * w + next] - in[size_t(y) * w + prev]) * 0.5f;
    }
}
void derivative_y(const std::vector<float>& in, int w, int h, std::vector<float>& out) {
  out.resize(size_t(w) * h);
  for (int y = 0; y < h; ++y) {
    int prev = y - 1 < 0 ? 0 : y - 1;
    int next = y + 1 > h - 1 ? h - 1 : y + 1;
    for (int x = 0; x < w; ++x)
      out[size_t(y) * w + x] = (in[size_t(next) * w + x] - in[size_t(prev) * w + x]) * 0.5f;
  }
}

void build_derivatives(Level& L) {
  derivative_x(L.ch[0], L.w, L.h, L.ch[2]);
  derivative_y(L.ch[0], L.w, L.h, L.ch[3]);
  derivative_x(L.ch[1], L.w, L.h, L.ch[4]);
  derivative_y(L.ch[1], L.w, L.h, L.ch[5]);
}

// ------------------------------------------------------------------------------------------
// SE(3): restated from the published Sophus (templated se3.hpp / so3.hpp, 2013) algorithm.
// Sophus is an un-vendored, unpinned dependency of the reference (sophus/Makefile:5-9);
// call sites: dense_tracking.cpp:147,238,259-261,302,346,371.
// ------------------------------------------------------------------------------------------
const double kSophusEps = 1e-10;

struct Quat { double w, x, y, z; };
struct SE3 {
  Quat q{1, 0, 0, 0};
  double t[3]{0, 0, 0};
};

Quat qmul(const Quat& a, const Quat& b) {
  return Quat{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z,
              a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
              a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
              a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
void qnormalize(Quat& q) {
  double n = std::sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  q.w /= n; q.x /= n; q.y /= n; q.z /= n;
}
void qrot(const Quat& q, double R[9]) {  // Eigen Quaternion::toRotationMatrix
  double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
Quat quat_from_rot(const double R[9]) {  // Eigen quaternion-from-matrix (Shepperd)
  Quat q;
  double tr = R[0] + R[4] + R[8];
  if (tr > 0) {
    double t = std::sqrt(tr + 1.0);
    q.w = 0.5 * t;
    t = 0.5 / t;
    q.x = (R[7] - R[5]) * t; q.y = (R[2] - R[6]) * t; q.z = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[i * 4]) i = 2;
    int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = std::sqrt(R[i * 4] - R[j * 4] - R[k * 4] + 1.0);
    double v[3];
    v[i] = 0.5 * t;
    t = 0.5 / t;
    q.w = (R[k * 3 + j] - R[j * 3 + k]) * t;
    v[j] = (R[j * 3 + i] + R[i * 3 + j]) * t;
    v[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
    q.x = v[0]; q.y = v[1]; q.z = v[2];
  }
  qnormalize(q);
  return q;
}

SE3 se3_mul(const SE3& a, const SE3& b) {
  SE3 r;
  r.q = qmul(a.q, b.q);
  qnormalize(r.q);
  double R[9];
  qrot(a.q, R);
  for (int i = 0; i < 3; ++i) r.t[i] = a.t[i] + R[i * 3 + 0] * b.t[0] + R[i * 3 + 1] * b.t[1] + R[i * 3 + 2] * b.t[2];
  return r;
}
SE3 se3_inverse(const SE3& a) {
  SE3 r;
  r.q = Quat{a.q.w, -a.q.x, -a.q.y, -a.q.z};
  double R[9];
  qrot(r.q, R);
  for (int i = 0; i < 3; ++i) r.t[i] = -(R[i * 3 + 0] * a.t[0] + R[i * 3 + 1] * a.t[1] + R[i * 3 + 2] * a.t[2]);
  return r;
}
void se3_matrix(const SE3& a, double T[16]) {
  double R[9];
  qrot(a.q, R);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[i * 4 + j] = R[i * 3 + j];
    T[i * 4 + 3] = a.t[i];
  }
  T[12] = T[13] = T[14] = 0;
  T[15] = 1;
}
SE3 se3_from_matrix(const double T[16]) {
  double R[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = T[i * 4 + j];
  SE3 r;
  r.q = quat_from_rot(R);
  for (int i = 0; i < 3; ++i) r.t[i] = T[i * 4 + 3];
  return r;
}
void hat(const double w[3], double O[9]) {
  O[0] = 0; O[1] = -w[2]; O[2] = w[1];
  O[3] = w[2]; O[4] = 0; O[5] = -w[0];
  O[6] = -w[1]; O[7] = w[0]; O[8] = 0;
}
void mat3mul(const double A[9], const double B[9], double C[9]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}
// SE3Group::exp: twist ordering [upsilon; omega]
SE3 se3_exp(const double a[6]) {
  const double* ups = a;
  const double* om = a + 3;
  double theta = std::sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
  double half = 0.5 * theta, imag, real;
  if (theta < kSophusEps) {
    double t2 = theta * theta, t4 = t2 * t2;
    imag = 0.5 - t2 / 48.0 + t4 / 3840.0;
    real = 1.0 - t2 / 8.0 + t4 / 384.0;
  } else {
    imag = std::sin(half) / theta;
    real = std::cos(half);
  }
  SE3 r;
  r.q = Quat{real, imag * om[0], imag * om[1], imag * om[2]};
  double O[9], O2[9], V[9];
  hat(om, O);
  mat3mul(O, O, O2);
  if (theta < kSophusEps) {
    qrot(r.q, V);
  } else {
    double t2 = theta * theta;
    double c1 = (1 - std::cos(theta)) / t2, c2 = (theta - std::sin(theta)) / (t2 * theta);
    for (int i = 0; i < 9; ++i) V[i] = c1 * O[i] + c2 * O2[i];
    V[0] += 1; V[4] += 1; V[8] += 1;
  }
  for (int i = 0; i < 3; ++i) r.t[i] = V[i * 3] * ups[0] + V[i * 3 + 1] * ups[1] + V[i * 3 + 2] * ups[2];
  return r;
}
// SE3Group::log
void se3_log(const SE3& s, double out[6]) {
  double sq = s.q.x * s.q.x + s.q.y * s.q.y + s.q.z * s.q.z;
  double n = std::sqrt(sq), w = s.q.w, two_atan;
  if (n < kSophusEps) {
    two_atan = 2.0 / w - 2.0 * sq / (w * w * w);
  } else if (std::fabs(w) < kSophusEps) {
    two_atan = (w > 0 ? M_PI : -M_PI) / n;
  } else {
    two_atan = 2.0 * std::atan(n / w) / n;
  }
  double theta = two_atan * n;
  double om[3] = {two_atan * s.q.x, two_atan * s.q.y, two_atan * s.q.z};
  double O[9], O2[9], Vi[9];
  hat(om, O);
  mat3mul(O, O, O2);
  double c;
  if (std::fabs(theta) < kSophusEps) {
    c = 1.0 / 12.0;
  } else {
    double half = 0.5 * theta;
    c = (1 - theta * std::cos(half) / (2 * std::sin(half))) / (theta * theta);
  }
  for (int i = 0; i < 9; ++i) Vi[i] = -0.5 * O[i] + c * O2[i];
  Vi[0] += 1; Vi[4] += 1; Vi[8] += 1;
  for (int i = 0; i < 3; ++i) out[i] = Vi[i * 3] * s.t[0] + Vi[i * 3 + 1] * s.t[1] + Vi[i * 3 + 2] * s.t[2];
  out[3] = om[0]; out[4] = om[1]; out[5] = om[2];
}

// dvo/util/revertable.h:45-55
template <typename T>
struct Revertable {
  T old, value;
  T& update() { old = value; return value; }
  void revert() { value = old; }
};

// ------------------------------------------------------------------------------------------
// n x n LDLT, n <= 8 (Eigen::LDLT restated: diagonal pivoting, in-place, then solve with the
// tolerance rule for D).  dense_tracking.cpp:347  x = A.ldlt().solve(b); n = 8 in the photometric mode.
// ------------------------------------------------------------------------------------------
void ldlt_solve(const double* Ain, const double* bin, double* x, int n) {
  double A[64];
  std::memcpy(A, Ain, sizeof(double) * n * n);
  int perm[8];
  for (int k = 0; k < n; ++k) {
    int piv = k;
    double best = std::fabs(A[k * n + k]);
    for (int i = k + 1; i < n; ++i)
      if (std::fabs(A[i * n + i]) > best) { best = std::fabs(A[i * n + i]); piv = i; }
    perm[k] = piv;
    if (piv != k) {  // symmetric row/col swap of the full matrix
      for (int j = 0; j < n; ++j) std::swap(A[k * n + j], A[piv * n + j]);
      for (int i = 0; i < n; ++i) std::swap(A[i * n + k], A[i * n + piv]);
    }
    // A[k][k] -= sum_j L[k][j]^2 D[j]; stored: lower part holds L, diagonal holds D
    for (int j = 0; j < k; ++j) A[k * n + k] -= A[k * n + j] * A[k * n + j] * A[j * n + j];
    double d = A[k * n + k];
    for (int i = k + 1; i < n; ++i) {
      double s = A[i * n + k];
      for (int j = 0; j < k; ++j) s -= A[i * n + j] * A[k * n + j] * A[j * n + j];
      A[i * n + k] = (d != 0.0) ? s / d : 0.0;
    }
  }
  double y[8];
  for (int i = 0; i < n; ++i) y[i] = bin[i];
  for (int k = 0; k < n; ++k) std::swap(y[k], y[perm[k]]);  // P b
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j) y[i] -= A[i * n + j] * y[j];  // L^-1
  double dmax = 0;
  for (int i = 0; i < n; ++i) dmax = std::fmax(dmax, std::fabs(A[i * n + i]));
  double tol = std::fmax(dmax * DBL_EPSILON, 1.0 / DBL_MAX);
  for (int i = 0; i < n; ++i) y[i] = std::fabs(A[i * n + i]) > tol ? y[i] / A[i * n + i] : 0.0;  // D^-1
  for (int i = n - 1; i >= 0; --i)
    for (int j = i + 1; j < n; ++j) y[i] -= A[j * n + i] * y[j];  // L^-T
  for (int k = n - 1; k >= 0; --k) std::swap(y[k], y[perm[k]]);  // P^T
  for (int i = 0; i < n; ++i) x[i] = y[i];
}
void ldlt_solve6(const double A[36], const double b[6], double x[6]) { ldlt_solve(A, b, x, 6); }

// A_xx - A_xp A_pp^-1 A_px of an 8 x 8 onto its first 6 unknowns, fp64, the 2 x 2 inverse written out
void schur_onto_pose(const double A[64], double S[36]) {
  const double a = A[6 * 8 + 6], c = A[6 * 8 + 7], d = A[7 * 8 + 7];
  const double rdet = 1.0 / (a * d - c * c);
  const double i00 = d * rdet, i01 = -c * rdet, i11 = a * rdet;
  for (int i = 0; i < 6; ++i) {
    const double g0 = i00 * A[i * 8 + 6] + i01 * A[i * 8 + 7], g1 = i01 * A[i * 8 + 6] + i11 * A[i * 8 + 7];
    for (int j = 0; j < 6; ++j) S[i * 6 + j] = A[i * 8 + j] - (g0 * A[j * 8 + 6] + g1 * A[j * 8 + 7]);
  }
}

// The motion prior Lambda (6 x 6, row-major) in place of mu I: s_i = sum_j Lambda_ij li_j in order j = 0..5 from 0, and the
// prior log-likelihood sum_i li_i s_i.  With -ffp-contract=off and Lambda = mu I every term but mu li_i is an exact zero, so
// b_i + s_i is the mu path's b_i + mu li_i; the log-likelihood rounds differently from mu |li|^2.
struct MotionPriorTerms {
  double s[6];   // Lambda li
  double ll;     // li^T Lambda li
};

MotionPriorTerms motion_prior_terms(const double L[36], const double li[6]) {
  MotionPriorTerms t;
  t.ll = 0.0;
  for (int i = 0; i < 6; ++i) {
    double s = 0.0;
    for (int j = 0; j < 6; ++j) s += L[i * 6 + j] * li[j];
    t.s[i] = s;
  }
  for (int i = 0; i < 6; ++i) t.ll += li[i] * t.s[i];
  return t;
}

// ------------------------------------------------------------------------------------------
// reference point list: PointWithIntensityAndDepth (rgbd_image.h:39-89), 48 bytes
// ------------------------------------------------------------------------------------------
struct RefPoint {
  float x, y, z, one;
  float i, zr, idx, idy, zdx, zdy, t0, t1;
  int pix;  // linear pixel index (not in the reference; used for the dense image outputs)
};

// PointSelection::selectPointsFromImage (point_selection.cpp:119-152) with
// ValidPointAndGradientThresholdPredicate::isPointOk (point_selection.h:63-66) and the point
// cloud of RgbdCamera ctor / buildPointCloud (rgbd_image.cpp:186-204, 245-262).
void select_points(const Level& L, float ti, float td, std::vector<RefPoint>& pts) {
  pts.clear();
  pts.reserve(size_t(L.w) * L.h);
  for (int y = 0; y < L.h; ++y)
    for (int x = 0; x < L.w; ++x) {
      size_t p = size_t(y) * L.w + x;
      float z = L.ch[1][p], idx = L.ch[2][p], idy = L.ch[3][p], zdx = L.ch[4][p], zdy = L.ch[5][p];
      bool ok = z == z && zdx == zdx && zdy == zdy &&
                (std::fabs(idx) > ti || std::fabs(idy) > ti || std::fabs(zdx) > td || std::fabs(zdy) > td);
      if (!ok) continue;
      RefPoint r;
      float tx = (float(x) - L.ox) / L.fx;  // pointcloud_template_ (rgbd_image.cpp:197-198)
      float ty = (float(y) - L.oy) / L.fy;
      r.x = tx * z; r.y = ty * z; r.z = 1.0f * z; r.one = 1.0f;  // rgbd_image.cpp:258-259
      r.i = L.ch[0][p]; r.zr = z; r.idx = idx; r.idy = idy; r.zdx = zdx; r.zdy = zdy; r.t0 = 0; r.t1 = 0;
      r.pix = int(p);
      pts.push_back(r);
    }
}

// The photometric mode (include/dvo_b200.h): the reference intensity of every selected point becomes alpha I_ref + beta
// before the residual loop, rounded to nearest, with (alpha, beta) as float.  At (1, 0) that is I_ref exactly.
void brighten_selection(std::vector<RefPoint>& pts, const double ab[2], const orc_mode& mode) {
  const float a = float(ab[0]), b = float(ab[1]);
  for (RefPoint& p : pts) p.i = mode.fused_pixel_math ? std::fmaf(a, p.i, b) : a * p.i + b;
}

struct ErrPoint {  // points_error entry: untransformed point + residual record (dense_tracking_impl.cpp:265-281)
  float x, y, z;
  float e[6];  // e.i, e.z, e.idx, e.idy, e.zdx, e.zdy
  int pix;
};

inline float rcp_ss(float v) { return _mm_cvtss_f32(_mm_rcp_ss(_mm_set_ss(v))); }

// depthStdDevZ (dense_tracking_impl.cpp:122-128)
inline float depth_std_dev_z(float depth) {
  float s = depth - 0.4f;
  s = 0.0012f + 0.0019f * s * s;
  return s;
}

struct LevelConsts {
  float kt[3][4];
  float wcur[6], wref[6];
  float ub_x, ub_y;
};

// KT = K * T[0:3,:] in float (dense_tracking_impl.cpp:142-152), wcur / wref (dense_tracking.cpp:215-220)
void make_level_consts(const Level& L, const double T[16], LevelConsts& c) {
  float Tf[3][4];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) Tf[i][j] = float(T[i * 4 + j]);  // dense_tracking.cpp:263 cast<float>
  for (int j = 0; j < 4; ++j) {
    // Eigen coefficient product: ((k0*t0 + k1*t1) + k2*t2); zero entries of K contribute exact 0
    c.kt[0][j] = (L.fx * Tf[0][j] + 0.0f * Tf[1][j]) + L.ox * Tf[2][j];
    c.kt[1][j] = (0.0f * Tf[0][j] + L.fy * Tf[1][j]) + L.oy * Tf[2][j];
    c.kt[2][j] = (0.0f * Tf[0][j] + 0.0f * Tf[1][j]) + 1.0f * Tf[2][j];
  }
  const float wcur_id = 0.5f, wref_id = 0.5f, wcur_zd = 1.0f, wref_zd = 0.0f;
  c.wcur[0] = 1.0f / 255.0f; c.wcur[1] = 1.0f;
  c.wcur[2] = wcur_id * L.fx / 255.0f; c.wcur[3] = wcur_id * L.fy / 255.0f;
  c.wcur[4] = wcur_zd * L.fx; c.wcur[5] = wcur_zd * L.fy;
  c.wref[0] = -1.0f / 255.0f; c.wref[1] = -1.0f;
  c.wref[2] = wref_id * L.fx / 255.0f; c.wref[3] = wref_id * L.fy / 255.0f;
  c.wref[4] = wref_zd * L.fx; c.wref[5] = wref_zd * L.fy;
  c.ub_x = float(L.w - 2); c.ub_y = float(L.h - 2);
}

// computeResidualsSse<false> (dense_tracking_impl.cpp:133-393), one point at a time; the SSE
// code processes two points per trip with identical per-lane arithmetic, so only the odd-point
// drop (line 169) is a pairwise effect.
// Unfused (reference) arithmetic.  Runs under RTZ when mode.rtz_residuals.
int64_t compute_residuals(const std::vector<RefPoint>& pts, const Level& cur, const LevelConsts& c,
                          const orc_mode& mode, std::vector<ErrPoint>& out) {
  out.clear();
  size_t S = pts.size();
  if (mode.drop_odd_point && (S % 2) != 0) S -= 1;
  unsigned int rnd = _MM_GET_ROUNDING_MODE();
  if (mode.rtz_residuals) _MM_SET_ROUNDING_MODE(_MM_ROUND_TOWARD_ZERO);
  const int W = cur.w;
  for (size_t k = 0; k < S; ++k) {
    const RefPoint& p = pts[k];
    float X, Y, Zt, u, v;
    int u0, v0;
    float fu, fv, gu, gv;
    float a[6];
    bool ok = true;
    if (!mode.fused_pixel_math) {
      // hadd(hadd(kt_r1*p, ...)) : (k0*x + k1*y) + (k2*z + k3*1)
      X = (c.kt[0][0] * p.x + c.kt[0][1] * p.y) + (c.kt[0][2] * p.z + c.kt[0][3] * p.one);
      Y = (c.kt[1][0] * p.x + c.kt[1][1] * p.y) + (c.kt[1][2] * p.z + c.kt[1][3] * p.one);
      Zt = (c.kt[2][0] * p.x + c.kt[2][1] * p.y) + (c.kt[2][2] * p.z + c.kt[2][3] * p.one);
      float r = mode.rcp_approx ? rcp_ss(Zt) : 1.0f / Zt;  // line 192
      u = X * r; v = Y * r;
    } else {
      // MIRROR of the CUDA kernel (dvo_slam_b200/csrc/pixel_math.cuh): fma chains + IEEE rcp
      X = std::fmaf(c.kt[0][0], p.x, std::fmaf(c.kt[0][1], p.y, std::fmaf(c.kt[0][2], p.z, c.kt[0][3])));
      Y = std::fmaf(c.kt[1][0], p.x, std::fmaf(c.kt[1][1], p.y, std::fmaf(c.kt[1][2], p.z, c.kt[1][3])));
      Zt = std::fmaf(c.kt[2][0], p.x, std::fmaf(c.kt[2][1], p.y, std::fmaf(c.kt[2][2], p.z, c.kt[2][3])));
      float r = 1.0f / Zt;
      u = X * r; v = Y * r;
    }
    // bounds: 0 <= u <= w-2, 0 <= v <= h-2 (lines 160-161, 203); NaN compares false
    if (!(u >= 0.0f && u <= c.ub_x && v >= 0.0f && v <= c.ub_y)) continue;
    u0 = int(u); v0 = int(v);  // cvtps_epi32 under RTZ == truncation (lines 165-167, 195)
    fu = u - float(u0); fv = v - float(v0);
    gu = 1.0f - fu; gv = 1.0f - fv;
    size_t i00 = size_t(v0) * W + u0, i10 = i00 + 1, i01 = i00 + W, i11 = i01 + 1;
    for (int ch = 0; ch < 6; ++ch) {
      const float* P = cur.ch[ch].data();
      if (!mode.fused_pixel_math)
        a[ch] = (gv * (gu * P[i00] + fu * P[i10])) + (fv * (gu * P[i01] + fu * P[i11]));  // lines 227-258
      else
        a[ch] = std::fmaf(fv, std::fmaf(fu, P[i11], gu * P[i01]), gv * std::fmaf(fu, P[i10], gu * P[i00]));
      if (a[ch] != a[ch]) ok = false;  // cmpunord over all lanes (line 261)
    }
    if (!ok) continue;
    ErrPoint e;
    e.x = p.x; e.y = p.y; e.z = p.z; e.pix = p.pix;
    if (!mode.fused_pixel_math) {
      e.e[0] = c.wcur[0] * a[0] + c.wref[0] * p.i;
      e.e[1] = c.wcur[1] * a[1] + c.wref[1] * Zt;  // reference depth replaced by transformed z (line 269)
      // occlusion test (line 275)
      if (!(e.e[1] > -20.0f * depth_std_dev_z(p.zr))) continue;
      e.e[2] = c.wcur[2] * a[2] + c.wref[2] * p.idx;
      e.e[3] = c.wcur[3] * a[3] + c.wref[3] * p.idy;
      e.e[4] = c.wcur[4] * a[4] + c.wref[4] * p.zdx;
      e.e[5] = c.wcur[5] * a[5] + c.wref[5] * p.zdy;
    } else {
      e.e[0] = std::fmaf(c.wcur[0], a[0], c.wref[0] * p.i);
      e.e[1] = a[1] - Zt;
      float s = p.zr - 0.4f;
      float sig = std::fmaf(0.0019f * s, s, 0.0012f);
      if (!(e.e[1] > -20.0f * sig)) continue;
      e.e[2] = std::fmaf(c.wcur[2], a[2], c.wref[2] * p.idx);
      e.e[3] = std::fmaf(c.wcur[3], a[3], c.wref[3] * p.idy);
      e.e[4] = c.wcur[4] * a[4];
      e.e[5] = c.wcur[5] * a[5];
    }
    out.push_back(e);
  }
  if (mode.rtz_residuals) _MM_SET_ROUNDING_MODE(rnd);
  return int64_t(out.size());
}

// computeWeight / computeWeightsSse (dense_tracking_impl.cpp:640-707), mean == 0 (dense_tracking.cpp:205)
void compute_weights(const std::vector<ErrPoint>& e, const float P[4] /*row-major*/, const orc_mode& mode,
                     std::vector<float>& w) {
  size_t n = e.size();
  w.resize(n);
  size_t n4 = mode.rcp_approx ? n - (n % 4) : 0;
  // prec = [P00, P10, P01, P11] (column-major load); dist = (x*P00 + y*P10)*x + (x*P01 + y*P11)*y
  for (size_t k = 0; k < n; ++k) {
    float x = e[k].e[0], y = e[k].e[1];
    float d = (x * P[0] + y * P[2]) * x + (x * P[1] + y * P[3]) * y;
    if (k < n4)
      w[k] = 7.0f * rcp_ss(5.0f + d);
    else
      w[k] = float((2.0 + 5.0f) / double(5.0f + d));
  }
}

// computeScale / computeScaleSse (dense_tracking_impl.cpp:566-638).  Returns covariance (row-major).
void compute_scale(const std::vector<ErrPoint>& e, const std::vector<float>& w, const orc_mode& mode, float C[4]) {
  size_t n = e.size();
  if (mode.f32_serial_accum) {
    float scale = 1.0f / float(n - 2 - 1);
    float acc[4] = {0, 0, 0, 0};
    size_t n2 = n - (n % 2);
    for (size_t k = 0; k < n2; k += 2) {
      float x1 = e[k].e[0], y1 = e[k].e[1];
      float x2 = mode.scale_pair_bug ? x1 : e[k + 1].e[0];  // lines 614-615 reuse the low half
      float y2 = mode.scale_pair_bug ? y1 : e[k + 1].e[1];
      float f1[4] = {x1 * x1, y1 * x1, x1 * y1, y1 * y1};
      float f2[4] = {x2 * x2, y2 * x2, x2 * y2, y2 * y2};
      for (int j = 0; j < 4; ++j) {
        float p1 = scale * (w[k] * f1[j]);
        float p2 = scale * (w[k + 1] * f2[j]);
        acc[j] = acc[j] + (p1 + p2);
      }
    }
    C[0] = acc[0]; C[1] = acc[1]; C[2] = acc[1]; C[3] = acc[3];
    for (size_t k = n2; k < n; ++k) {  // scalar tail: covariance += scale * (weight*diff)*diff^T
      float x = e[k].e[0], y = e[k].e[1];
      float wx = w[k] * x, wy = w[k] * y;
      C[0] += scale * (wx * x); C[1] += scale * (wx * y);
      C[2] += scale * (wy * x); C[3] += scale * (wy * y);
    }
  } else {
    double acc[3] = {0, 0, 0};
    size_t n2 = n - (n % 2);
    for (size_t k = 0; k < n; ++k) {
      size_t src = k;
      if (mode.scale_pair_bug && k < n2 && (k & 1)) src = k - 1;  // follower reuses the leader's residual
      double x = e[src].e[0], y = e[src].e[1], ww = w[k];
      acc[0] += ww * x * x; acc[1] += ww * x * y; acc[2] += ww * y * y;
    }
    double s = 1.0 / double(n - 3);
    C[0] = float(acc[0] * s); C[1] = float(acc[1] * s); C[2] = C[1]; C[3] = float(acc[2] * s);
  }
}

// Eigen Matrix2f::inverse (dense_tracking.cpp:295)
void inverse2(const float C[4], float P[4]) {
  float det = C[0] * C[3] - C[1] * C[2];
  float invdet = 1.0f / det;
  P[0] = C[3] * invdet; P[1] = -C[1] * invdet; P[2] = -C[2] * invdet; P[3] = C[0] * invdet;
}

// computeCompleteDataLogLikelihood (dense_tracking_impl.cpp:406-425)
float compute_ll(const std::vector<ErrPoint>& e, const float P[4], const orc_mode& mode) {
  size_t n = e.size();
  double error_sum = 0.0, error_acc = 1.0;
  size_t c = 1;
  for (size_t k = 0; k < n; ++k, ++c) {
    float x = e[k].e[0], y = e[k].e[1];
    float d = (x * P[0] + y * P[2]) * x + (x * P[1] + y * P[3]) * y;  // r^T P r in float
    if (!mode.ll_group_product) {   // the per-point logs summed; ll_drop_tail still drops the last n % 50
      if (!mode.ll_drop_tail || k < n - n % 50) error_sum += std::log(1.0 + 0.2 * double(d));
      continue;
    }
    error_acc *= (1.0 + 0.2 * double(d));
    if ((c % 50) == 0) {
      error_sum += std::log(error_acc);
      error_acc = 1.0;
    }
  }
  if (mode.ll_group_product && !mode.ll_drop_tail) error_sum += std::log(error_acc);
  float det = P[0] * P[3] - P[1] * P[2];
  return float(0.5 * double(n) * double(std::log(det)) - 0.5 * (5.0 + 2.0) * error_sum);
}

// Jacobians (dense_tracking.cpp:448-476) + row assembly (dense_tracking.cpp:338-339)
template <typename F>
void jacobian_rows(F x, F y, F z, F idx, F idy, F zdx, F zdy, F J0[6], F J1[6]) {
  F zi = F(1) / z, zs = F(1) / (z * z);
  F Jw0[6], Jw1[6];
  Jw0[0] = zi; Jw0[1] = 0; Jw0[2] = -x * zs; Jw0[3] = Jw0[2] * y; Jw0[4] = F(1) - Jw0[2] * x; Jw0[5] = -y * zi;
  Jw1[0] = 0; Jw1[1] = zi; Jw1[2] = -y * zs; Jw1[3] = F(-1) + Jw1[2] * y; Jw1[4] = -Jw0[3]; Jw1[5] = x * zi;
  F Jz[6] = {0, 0, 1, y, -x, 0};
  for (int c = 0; c < 6; ++c) {
    J0[c] = idx * Jw0[c] + idy * Jw1[c];
    J1[c] = (zdx * Jw0[c] + zdy * Jw1[c]) - Jz[c];
  }
}

// NormalEquationsLeastSquares::update(2x6 J, 2 r, 2x2 W) (least_squares.cpp:58-64) via
// OptimizedSelfAdjointMatrix6x6f::rankUpdate (math_sse.cpp:82-178), toEigen (math_sse.cpp:190-207).
void normal_equations(const std::vector<ErrPoint>& e, const std::vector<float>& w, const float P[4],
                      const orc_mode& mode, double A[36], double b[6]) {
  size_t n = e.size();
  if (mode.f32_serial_accum) {
    float blk[6][4];  // blocks (0,0) (0,2) (0,4) (2,2) (2,4) (4,4), each row-major 2x2
    float bf[6] = {0, 0, 0, 0, 0, 0};
    std::memset(blk, 0, sizeof(blk));
    for (size_t k = 0; k < n; ++k) {
      float J0[6], J1[6];
      jacobian_rows<float>(e[k].x, e[k].y, e[k].z, e[k].e[2], e[k].e[3], e[k].e[4], e[k].e[5], J0, J1);
      float W[4] = {w[k] * P[0], w[k] * P[1], w[k] * P[2], w[k] * P[3]};  // (*w_it) * precision
      // u_a(c) = v_a*W00 + v_b*W10 ; u_b(c) = v_a*W01 + v_b*W11
      float ua[6], ub[6];
      for (int c = 0; c < 6; ++c) {
        ua[c] = J0[c] * W[0] + J1[c] * W[2];
        ub[c] = J0[c] * W[1] + J1[c] * W[3];
      }
      static const int bi[6] = {0, 0, 0, 2, 2, 4}, bj[6] = {0, 2, 4, 2, 4, 4};
      for (int q = 0; q < 6; ++q) {
        int i = bi[q], j = bj[q];
        blk[q][0] += ua[i] * J0[j] + ub[i] * J1[j];
        blk[q][1] += ua[i] * J0[j + 1] + ub[i] * J1[j + 1];
        blk[q][2] += ua[i + 1] * J0[j] + ub[i + 1] * J1[j];
        blk[q][3] += ua[i + 1] * J0[j + 1] + ub[i + 1] * J1[j + 1];
      }
      // b -= J^T * W * r : (J^T W)(i,c) = J0[i]*W(0,c) + J1[i]*W(1,c); then * r
      float r0 = e[k].e[0], r1 = e[k].e[1];
      for (int i = 0; i < 6; ++i) {
        float m0 = J0[i] * W[0] + J1[i] * W[2];
        float m1 = J0[i] * W[1] + J1[i] * W[3];
        bf[i] -= m0 * r0 + m1 * r1;
      }
    }
    float Af[36];
    std::memset(Af, 0, sizeof(Af));
    static const int bi[6] = {0, 0, 0, 2, 2, 4}, bj[6] = {0, 2, 4, 2, 4, 4};
    for (int q = 0; q < 6; ++q) {
      int i = bi[q], j = bj[q];
      Af[i * 6 + j] = blk[q][0]; Af[i * 6 + j + 1] = blk[q][1];
      Af[(i + 1) * 6 + j] = blk[q][2]; Af[(i + 1) * 6 + j + 1] = blk[q][3];
    }
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) A[i * 6 + j] = double(i <= j ? Af[i * 6 + j] : Af[j * 6 + i]);  // selfadjointView<Upper>
    for (int i = 0; i < 6; ++i) b[i] = double(bf[i]);
  } else {
    double Ad[36], bd[6];
    std::memset(Ad, 0, sizeof(Ad));
    std::memset(bd, 0, sizeof(bd));
    for (size_t k = 0; k < n; ++k) {
      float J0[6], J1[6];
      jacobian_rows<float>(e[k].x, e[k].y, e[k].z, e[k].e[2], e[k].e[3], e[k].e[4], e[k].e[5], J0, J1);
      double W[4] = {double(w[k]) * P[0], double(w[k]) * P[1], double(w[k]) * P[2], double(w[k]) * P[3]};
      double r0 = e[k].e[0], r1 = e[k].e[1];
      for (int i = 0; i < 6; ++i) {
        double ua = J0[i] * W[0] + J1[i] * W[2], ub = J0[i] * W[1] + J1[i] * W[3];
        for (int j = i; j < 6; ++j) Ad[i * 6 + j] += ua * J0[j] + ub * J1[j];
        bd[i] -= ua * r0 + ub * r1;
      }
    }
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) A[i * 6 + j] = i <= j ? Ad[i * 6 + j] : Ad[j * 6 + i];
    for (int i = 0; i < 6; ++i) b[i] = bd[i];
  }
}

// The photometric mode's 8 x 8: the per-entry arithmetic of normal_equations over the Jacobian rows extended by
// de_i/dalpha = -I_ref/255, de_i/dbeta = -1/255 (intensity row) and zeros (depth row), I_ref read from the reference level
// R; f32_serial_accum: fp32 in point order (the pose block equals the default FAITHFUL A and b bit for bit), else fp64.
void normal_equations_photometric(const std::vector<ErrPoint>& e, const std::vector<float>& w, const float P[4], const Level& R,
                       const orc_mode& mode, double A[64], double b[8]) {
  const float wref0 = -1.0f / 255.0f;
  const size_t n = e.size();
  float Af[64] = {0}, bf[8] = {0};
  double Ad[64] = {0}, bd[8] = {0};
  for (size_t k = 0; k < n; ++k) {
    float J0[8], J1[8];
    jacobian_rows<float>(e[k].x, e[k].y, e[k].z, e[k].e[2], e[k].e[3], e[k].e[4], e[k].e[5], J0, J1);
    J0[6] = wref0 * R.ch[0][size_t(e[k].pix)]; J0[7] = wref0;
    J1[6] = 0.0f; J1[7] = 0.0f;
    if (mode.f32_serial_accum) {
      const float W[4] = {w[k] * P[0], w[k] * P[1], w[k] * P[2], w[k] * P[3]};
      const float r0 = e[k].e[0], r1 = e[k].e[1];
      for (int i = 0; i < 8; ++i) {
        const float ua = J0[i] * W[0] + J1[i] * W[2], ub = J0[i] * W[1] + J1[i] * W[3];
        for (int j = i; j < 8; ++j) Af[i * 8 + j] += ua * J0[j] + ub * J1[j];
        bf[i] -= ua * r0 + ub * r1;
      }
    } else {
      const double W[4] = {double(w[k]) * P[0], double(w[k]) * P[1], double(w[k]) * P[2], double(w[k]) * P[3]};
      const double r0 = e[k].e[0], r1 = e[k].e[1];
      for (int i = 0; i < 8; ++i) {
        const double ua = J0[i] * W[0] + J1[i] * W[2], ub = J0[i] * W[1] + J1[i] * W[3];
        for (int j = i; j < 8; ++j) Ad[i * 8 + j] += ua * J0[j] + ub * J1[j];
        bd[i] -= ua * r0 + ub * r1;
      }
    }
  }
  for (int i = 0; i < 8; ++i)
    for (int j = 0; j < 8; ++j) {
      const int u = i <= j ? i * 8 + j : j * 8 + i;
      A[i * 8 + j] = mode.f32_serial_accum ? double(Af[u]) : Ad[u];
    }
  for (int i = 0; i < 8; ++i) b[i] = mode.f32_serial_accum ? double(bf[i]) : bd[i];
}

double linf6(const double x[6]) {
  double m = 0;
  for (int i = 0; i < 6; ++i) m = std::fmax(m, std::fabs(x[i]));
  // lpNorm<Infinity> of a vector containing NaN: Eigen's maxCoeff ignores/propagates inconsistently;
  // here NaN propagates so that "x > precision" is false, like a NaN comparison in the reference.
  for (int i = 0; i < 6; ++i)
    if (x[i] != x[i]) return kNaN;
  return m;
}

int64_t max_points(const orc_pyramid* p, int level) {  // point_selection.cpp:68-71
  size_t total = size_t(p->levels[0].w) * p->levels[0].h;
  return int64_t(size_t(double(total) * std::pow(0.25, double(level))));
}

}  // namespace

// ==========================================================================================
// C API
// ==========================================================================================
extern "C" {

orc_mode orc_mode_faithful(void) { return orc_mode{1, 1, 1, 1, 1, 1, 0, 1}; }
orc_mode orc_mode_exact(void) { return orc_mode{0, 0, 0, 0, 0, 0, 0, 0}; }
orc_mode orc_mode_mirror(void) { return orc_mode{0, 0, 1, 1, 1, 0, 1, 1}; }

orc_config orc_config_default(void) {  // dense_tracking_config.cpp:27-42
  orc_config c;
  c.first_level = 3; c.last_level = 1; c.max_iterations_per_level = 100; c.precision = 5e-7;
  c.mu = 0; c.use_initial_estimate = 0; c.intensity_derivative_threshold = 0.0f; c.depth_derivative_threshold = 0.0f;
  return c;
}

orc_pyramid* orc_pyramid_create(const float* intensity, const float* depth, int width, int height,
                                float fx, float fy, float ox, float oy, int levels) {
  if (levels < 1 || levels > ORC_MAX_LEVELS) return nullptr;
  orc_pyramid* p = new orc_pyramid;
  p->levels.resize(levels);
  Level& L0 = p->levels[0];
  L0.w = width; L0.h = height; L0.fx = fx; L0.fy = fy; L0.ox = ox; L0.oy = oy;
  L0.ch[0].assign(intensity, intensity + size_t(width) * height);
  L0.ch[1].assign(depth, depth + size_t(width) * height);
  build_derivatives(L0);
  for (int l = 1; l < levels; ++l) {
    const Level& P = p->levels[l - 1];
    Level& L = p->levels[l];
    L.w = P.w / 2; L.h = P.h / 2;
    // IntrinsicMatrix::scale(0.5f): whole 3x3 times 0.5 (intrinsic_matrix.cpp:90-93, rgbd_image.cpp:283-296)
    L.fx = P.fx * 0.5f; L.fy = P.fy * 0.5f; L.ox = P.ox * 0.5f; L.oy = P.oy * 0.5f;
    pyr_down_mean(P.ch[0], P.w, P.h, L.ch[0]);
    pyr_down_subsample(P.ch[1], P.w, P.h, L.ch[1]);
    build_derivatives(L);
  }
  return p;
}
void orc_pyramid_destroy(orc_pyramid* p) { delete p; }
int orc_pyramid_num_levels(const orc_pyramid* p) { return int(p->levels.size()); }
const float* orc_pyramid_plane(const orc_pyramid* p, int level, int channel) { return p->levels[level].ch[channel].data(); }
void orc_pyramid_level_info(const orc_pyramid* p, int level, int* width, int* height, float K[4]) {
  const Level& L = p->levels[level];
  *width = L.w; *height = L.h;
  K[0] = L.fx; K[1] = L.fy; K[2] = L.ox; K[3] = L.oy;
}

int64_t orc_select(const orc_pyramid* ref, int level, float ti, float td, const orc_mode* mode, uint8_t* mask) {
  std::vector<RefPoint> pts;
  const Level& L = ref->levels[level];
  select_points(L, ti, td, pts);
  size_t S = pts.size();
  if (mask) {
    std::memset(mask, 0, size_t(L.w) * L.h);
    size_t used = (mode && mode->drop_odd_point && (S % 2)) ? S - 1 : S;
    for (size_t k = 0; k < used; ++k) mask[pts[k].pix] = 1;
  }
  return int64_t(S);
}

int64_t orc_residual_image(const orc_pyramid* ref, const orc_pyramid* cur, int level, const double T[16],
                           const double ab[2], float ti, float td, const orc_mode* mode, float* planes7) {
  const Level& R = ref->levels[level];
  const Level& C = cur->levels[level];
  std::vector<RefPoint> pts;
  select_points(R, ti, td, pts);
  if (ab) brighten_selection(pts, ab, *mode);
  LevelConsts c;
  make_level_consts(C, T, c);
  std::vector<ErrPoint> e;
  compute_residuals(pts, C, c, *mode, e);
  size_t N = size_t(R.w) * R.h;
  for (size_t i = 0; i < 7 * N; ++i) planes7[i] = kNaNf;
  for (const ErrPoint& q : e) {
    for (int k = 0; k < 6; ++k) planes7[size_t(k) * N + q.pix] = q.e[k];
    planes7[6 * N + q.pix] = q.z;
  }
  return int64_t(e.size());
}

// DenseTracker::computeIntensityErrorImage (dense_tracking.cpp:378-444): residuals with valid flags
// (computeResidualsAndValidFlagsSse), then a raster walk over the selection's debug index (1 at every
// selected pixel, point_selection.cpp:139-140) that consumes one valid flag per selected pixel and one
// residual per set flag.  The flag vector is zero-initialised (line 391) and the SSE loop never visits
// the odd last point (dense_tracking_impl.cpp:169), so that pixel reads flag 0 and stays 0 in the image.
int64_t orc_intensity_error_image(const orc_pyramid* ref, const orc_pyramid* cur, int level, const double T[16],
                                  float ti, float td, const orc_mode* mode, float* image) {
  const Level& R = ref->levels[level];
  const Level& C = cur->levels[level];
  std::vector<RefPoint> pts;
  select_points(R, ti, td, pts);
  LevelConsts c;
  make_level_consts(C, T, c);
  std::vector<ErrPoint> e;
  compute_residuals(pts, C, c, *mode, e);
  const size_t N = size_t(R.w) * R.h;
  std::vector<uint8_t> debug_idx(N, 0), valid(pts.size(), 0);
  for (const RefPoint& p : pts) debug_idx[size_t(p.pix)] = 1;
  {  // last_valid_flag stream: one flag per visited point, 1 iff the point produced a residual (lines 292-293, 388-389)
    size_t j = 0;
    for (size_t k = 0; k < pts.size() && j < e.size(); ++k)
      if (e[j].pix == pts[k].pix) { valid[k] = 1; ++j; }
  }
  for (size_t i = 0; i < N; ++i) image[i] = 0.0f;                    // cv::Mat::zeros (line 415)
  size_t flag_it = 0, res_it = 0;
  for (size_t i = 0; i < N; ++i) {                                   // lines 426-439
    if (debug_idx[i] == 1) {
      if (valid[flag_it] == 1) {
        image[i] = std::fabs(e[res_it].e[0]);
        ++res_it;
      }
      ++flag_it;
    }
  }
  return int64_t(res_it);
}

int64_t orc_linearize(const orc_pyramid* ref, const orc_pyramid* cur, int level, const double T[16], const double ab[2],
                      float ti, float td, int use_weights, const float prev_precision[4], const orc_mode* mode,
                      float precision_out[4], float* ll_out, double* A_out, double* b_out) {
  const Level& R = ref->levels[level];
  const Level& C = cur->levels[level];
  std::vector<RefPoint> pts;
  select_points(R, ti, td, pts);
  if (ab) brighten_selection(pts, ab, *mode);
  LevelConsts c;
  make_level_consts(C, T, c);
  std::vector<ErrPoint> e;
  int64_t n = compute_residuals(pts, C, c, *mode, e);
  if (n < 6) return n;
  std::vector<float> w;
  if (!use_weights) w.assign(size_t(n), 1.0f);
  else compute_weights(e, prev_precision, *mode, w);
  float Cov[4];
  compute_scale(e, w, *mode, Cov);
  inverse2(Cov, precision_out);
  *ll_out = compute_ll(e, precision_out, *mode);
  if (ab) normal_equations_photometric(e, w, precision_out, R, *mode, A_out, b_out);
  else normal_equations(e, w, precision_out, *mode, A_out, b_out);
  return n;
}

int orc_match_with(orc_pyramid* ref, orc_pyramid* cur, const orc_config* cfg, const double T_init[16], const double prior[36],
                   const double ab_init[2], const orc_mode* mode_p, orc_result* result, double ab_out[2],
                   orc_iteration_stats* iters, int max_iters, int* num_iters) {
  const orc_mode mode = *mode_p;
  const bool photometric = ab_out != nullptr;
  const int nu = photometric ? 8 : 6;  // unknowns: the pose, then (alpha, beta) in the photometric mode
  int iter_count = 0;
  std::memset(result, 0, sizeof(*result));

  // dense_tracking.cpp:137-147
  SE3 inc;
  if (cfg->use_initial_estimate) inc = se3_from_matrix(T_init);
  Revertable<SE3> initial{inc, inc};
  Revertable<SE3> estimate{SE3(), SE3()};
  // the photometric mode's (alpha, beta): updated and reverted with the pose, carried over between levels
  struct AB { double v[2]; };
  Revertable<AB> ab{{{1.0, 0.0}}, {{1.0, 0.0}}};
  if (ab_init) { ab.value.v[0] = ab.old.v[0] = ab_init[0]; ab.value.v[1] = ab.old.v[1] = ab_init[1]; }
  bool accept = true;

  float precision[4] = {0, 0, 0, 0};
  // per-thread scratch (the reference keeps points_error / residuals / weights as DenseTracker members, dense_tracking.cpp:160-165)
  // and pts_ab, the selection with the brightness model applied in the photometric mode
  static thread_local std::vector<RefPoint> pts, pts_ab;
  static thread_local std::vector<ErrPoint> err;
  static thread_local std::vector<float> weights;

  // per-level record of the last two iterations' information/LL for the final pick (lines 368-373)
  std::vector<orc_iteration_stats> level_iters;

  for (int level = cfg->first_level; level >= cfg->last_level; --level) {
    orc_level_stats& ls = result->levels[result->num_levels++];
    level_iters.clear();
    precision[0] = precision[1] = precision[2] = precision[3] = 0;  // line 206
    int iteration = 0;                                              // line 209
    double error = std::numeric_limits<double>::max(), last_error;  // line 210

    const Level& C = cur->levels[level];
    const Level& R = ref->levels[level];
    select_points(R, cfg->intensity_derivative_threshold, cfg->depth_derivative_threshold, pts);  // line 225

    ls.id = level;
    ls.max_valid_pixels = max_points(ref, level);
    ls.valid_pixels = int64_t(pts.size());
    ls.termination = -1;

    double A[64], b[8], x[8];
    se3_log(inc, x);  // line 238
    double dab[2] = {0.0, 0.0};  // the (alpha, beta) part of the last accepted increment of this level

    do {
      orc_iteration_stats it;
      std::memset(&it, 0, sizeof(it));
      for (int i = 0; i < 36; ++i) it.information[i] = kNaN;
      for (int i = 0; i < 6; ++i) it.increment[i] = kNaN;
      it.level = level;
      it.id = iteration;

      inc = se3_exp(x);                                             // line 259
      initial.update() = se3_mul(se3_inverse(inc), initial.value);  // line 260
      estimate.update() = se3_mul(inc, estimate.value);             // line 261
      if (photometric) {
        const AB prev = ab.value;
        ab.update() = AB{{prev.v[0] + dab[0], prev.v[1] + dab[1]}};
      }

      double T[16];
      se3_matrix(estimate.value, T);
      LevelConsts c;
      make_level_consts(C, T, c);
      if (photometric) {
        pts_ab = pts;
        brighten_selection(pts_ab, ab.value.v, mode);
      }
      int64_t n = compute_residuals(photometric ? pts_ab : pts, C, c, mode, err);  // line 271
      it.valid_constraints = n;

      if (n < 6) {                                                  // lines 276-284
        initial.revert();
        estimate.revert();
        if (photometric) ab.revert();
        ls.termination = ORC_TERM_TOO_FEW_CONSTRAINTS;
        level_iters.push_back(it);
        break;
      }
      if (iteration == 0) weights.assign(size_t(n), 1.0f);          // lines 286-293
      else compute_weights(err, precision, mode, weights);

      float Cov[4];
      compute_scale(err, weights, mode, Cov);                       // line 295
      inverse2(Cov, precision);
      float ll = compute_ll(err, precision, mode);                  // line 297

      it.tdist_log_likelihood = -double(ll);
      for (int i = 0; i < 4; ++i) it.tdist_precision[i] = double(precision[i]);
      double li[6];
      se3_log(initial.value, li);
      MotionPriorTerms pt;
      if (prior) {
        pt = motion_prior_terms(prior, li);
        it.prior_log_likelihood = pt.ll;
      } else {
        double sq = 0;
        for (int i = 0; i < 6; ++i) sq += li[i] * li[i];
        it.prior_log_likelihood = cfg->mu * sq;                     // line 302
      }

      last_error = error;                                           // lines 306-307
      error = -double(ll);
      accept = error < last_error;                                  // line 312
      if (!accept) {
        initial.revert();
        estimate.revert();
        if (photometric) ab.revert();
        ls.termination = ORC_TERM_LOG_LIKELIHOOD_DECREASED;
        level_iters.push_back(it);
        break;
      }

      if (photometric) normal_equations_photometric(err, weights, precision, R, mode, A, b);
      else normal_equations(err, weights, precision, mode, A, b);   // lines 333-343
      for (int i = 0; i < 6; ++i) {
        if (prior) {
          for (int j = 0; j < 6; ++j) A[i * nu + j] += prior[i * 6 + j];
          b[i] += pt.s[i];
        } else {
          A[i * nu + i] += cfg->mu;                                 // line 345
          b[i] += cfg->mu * li[i];                                  // line 346 (log of updated initial)
        }
      }
      ldlt_solve(A, b, x, nu);                                      // line 347
      for (int i = 0; i < 6; ++i) it.increment[i] = x[i];
      if (photometric) {
        dab[0] = x[6]; dab[1] = x[7];
        schur_onto_pose(A, it.information);
      } else {
        for (int i = 0; i < 36; ++i) it.information[i] = A[i];
      }
      level_iters.push_back(it);
      iteration++;                                                  // line 353
    } while (accept && linf6(x) > cfg->precision && !(iteration >= cfg->max_iterations_per_level));  // line 357

    if (linf6(x) <= cfg->precision) ls.termination = ORC_TERM_INCREMENT_TOO_SMALL;              // line 359
    if (iteration >= cfg->max_iterations_per_level) ls.termination = ORC_TERM_ITERATIONS_EXCEEDED;  // line 362
    ls.num_iterations = int32_t(level_iters.size());
    for (const orc_iteration_stats& it : level_iters) {
      if (iters && iter_count < max_iters) iters[iter_count] = it;
      iter_count++;
    }
  }

  // dense_tracking.cpp:368-373
  const orc_level_stats& last_level = result->levels[result->num_levels - 1];
  int pick = last_level.termination != ORC_TERM_LOG_LIKELIHOOD_DECREASED ? int(level_iters.size()) - 1
                                                                          : int(level_iters.size()) - 2;
  double Tm[16];
  se3_matrix(se3_inverse(estimate.value), Tm);
  std::memcpy(result->transformation, Tm, sizeof(Tm));
  if (pick >= 0) {
    for (int i = 0; i < 36; ++i) result->information[i] = level_iters[pick].information[i] * 0.008 * 0.008;
    result->log_likelihood = level_iters[pick].tdist_log_likelihood + level_iters[pick].prior_log_likelihood;
  } else {
    // reference reads out of bounds here (SURVEY Q24); defined behaviour: NaN so Result::isNaN() fires
    for (int i = 0; i < 36; ++i) result->information[i] = kNaN;
    result->log_likelihood = kNaN;
  }
  if (ab_out) { ab_out[0] = ab.value.v[0]; ab_out[1] = ab.value.v[1]; }
  if (num_iters) *num_iters = iter_count;
  return 0;
}

int orc_match(orc_pyramid* ref, orc_pyramid* cur, const orc_config* cfg, const double T_init[16],
              const orc_mode* mode, orc_result* result, orc_iteration_stats* iters, int max_iters,
              int* num_iters) {
  return orc_match_with(ref, cur, cfg, T_init, nullptr, nullptr, mode, result, nullptr, iters, max_iters, num_iters);
}

void orc_se3_exp(const double xi[6], double T[16]) { se3_matrix(se3_exp(xi), T); }
void orc_se3_log(const double T[16], double xi[6]) { se3_log(se3_from_matrix(T), xi); }
void orc_ldlt_solve6(const double A[36], const double b[6], double x[6]) { ldlt_solve6(A, b, x); }
void orc_ldlt_solve(const double* A, const double* b, double* x, int n) { ldlt_solve(A, b, x, n); }
void orc_schur_onto_pose(const double A[64], double S[36]) { schur_onto_pose(A, S); }

void orc_convert_raw_depth(const uint16_t* in, float* out, int64_t count, float scale) {
  for (int64_t i = 0; i < count; ++i) out[i] = in[i] == 0 ? kNaNf : float(in[i]) * scale;
}

void orc_bgr_to_grey(const uint8_t* bgr, float* out, int64_t count) {
  for (int64_t i = 0; i < count; ++i) {
    const int b = bgr[3 * i], g = bgr[3 * i + 1], r = bgr[3 * i + 2];
    out[i] = float((b * 1868 + g * 9617 + r * 4899 + (1 << 13)) >> 14);
  }
}

}  // extern "C"
