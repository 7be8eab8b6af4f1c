// se3.cuh -- SE(3) bookkeeping and the 6x6 solve of the Gauss-Newton step, fp64, usable on host and
// device.  Replaces the Sophus::SE3d / Eigen::LDLT calls of dvo::DenseTracker::match()
// (dvo_core/src/dense_tracking.cpp:147,238,259-261,302,346-347,371).  Sophus and Eigen are not
// vendored by the reference (sophus/Makefile:5-9); this follows their published closed forms:
// unit-quaternion rotation, twist order [v; omega], V-matrix exp/log, diagonal-pivoted LDL^T.
#pragma once
#include <cfloat>
#include <cmath>

#ifdef __CUDACC__
#define DVO_HD __host__ __device__ __forceinline__
#else
#define DVO_HD inline
#endif

namespace dvo_b200 {

struct SE3d {
  double qw, qx, qy, qz;  // unit quaternion
  double tx, ty, tz;
};

DVO_HD SE3d se3_identity() { return SE3d{1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0}; }

DVO_HD void se3_rotation(const SE3d& s, double R[9]) {
  double x2 = 2 * s.qx, y2 = 2 * s.qy, z2 = 2 * s.qz;
  double wx = x2 * s.qw, wy = y2 * s.qw, wz = z2 * s.qw;
  double xx = x2 * s.qx, xy = y2 * s.qx, xz = z2 * s.qx;
  double yy = y2 * s.qy, yz = z2 * s.qy, zz = z2 * s.qz;
  R[0] = 1 - (yy + zz); R[1] = xy - wz;       R[2] = xz + wy;
  R[3] = xy + wz;       R[4] = 1 - (xx + zz); R[5] = yz - wx;
  R[6] = xz - wy;       R[7] = yz + wx;       R[8] = 1 - (xx + yy);
}

DVO_HD void se3_normalize(SE3d& s) {
  double n = sqrt(s.qw * s.qw + s.qx * s.qx + s.qy * s.qy + s.qz * s.qz);
  double inv = 1.0 / n;
  s.qw *= inv; s.qx *= inv; s.qy *= inv; s.qz *= inv;
}

DVO_HD SE3d se3_mul(const SE3d& a, const SE3d& b) {
  SE3d r;
  r.qw = a.qw * b.qw - a.qx * b.qx - a.qy * b.qy - a.qz * b.qz;
  r.qx = a.qw * b.qx + a.qx * b.qw + a.qy * b.qz - a.qz * b.qy;
  r.qy = a.qw * b.qy - a.qx * b.qz + a.qy * b.qw + a.qz * b.qx;
  r.qz = a.qw * b.qz + a.qx * b.qy - a.qy * b.qx + a.qz * b.qw;
  se3_normalize(r);
  double R[9];
  se3_rotation(a, R);
  r.tx = a.tx + R[0] * b.tx + R[1] * b.ty + R[2] * b.tz;
  r.ty = a.ty + R[3] * b.tx + R[4] * b.ty + R[5] * b.tz;
  r.tz = a.tz + R[6] * b.tx + R[7] * b.ty + R[8] * b.tz;
  return r;
}

DVO_HD SE3d se3_inverse(const SE3d& a) {
  SE3d r;
  r.qw = a.qw; r.qx = -a.qx; r.qy = -a.qy; r.qz = -a.qz;
  double R[9];
  se3_rotation(r, R);
  r.tx = -(R[0] * a.tx + R[1] * a.ty + R[2] * a.tz);
  r.ty = -(R[3] * a.tx + R[4] * a.ty + R[5] * a.tz);
  r.tz = -(R[6] * a.tx + R[7] * a.ty + R[8] * a.tz);
  return r;
}

DVO_HD void se3_matrix(const SE3d& a, double T[16]) {
  double R[9];
  se3_rotation(a, R);
  T[0] = R[0]; T[1] = R[1]; T[2] = R[2];  T[3] = a.tx;
  T[4] = R[3]; T[5] = R[4]; T[6] = R[5];  T[7] = a.ty;
  T[8] = R[6]; T[9] = R[7]; T[10] = R[8]; T[11] = a.tz;
  T[12] = 0; T[13] = 0; T[14] = 0; T[15] = 1;
}

// rotation matrix -> unit quaternion (Shepperd's method), translation copied
DVO_HD SE3d se3_from_matrix(const double T[16]) {
  const double m00 = T[0], m01 = T[1], m02 = T[2], m10 = T[4], m11 = T[5], m12 = T[6], m20 = T[8], m21 = T[9], m22 = T[10];
  SE3d s;
  double tr = m00 + m11 + m22;
  if (tr > 0) {
    double t = sqrt(tr + 1.0);
    s.qw = 0.5 * t; t = 0.5 / t;
    s.qx = (m21 - m12) * t; s.qy = (m02 - m20) * t; s.qz = (m10 - m01) * t;
  } else if (m00 >= m11 && m00 >= m22) {
    double t = sqrt(m00 - m11 - m22 + 1.0);
    s.qx = 0.5 * t; t = 0.5 / t;
    s.qw = (m21 - m12) * t; s.qy = (m10 + m01) * t; s.qz = (m20 + m02) * t;
  } else if (m11 >= m22) {
    double t = sqrt(m11 - m22 - m00 + 1.0);
    s.qy = 0.5 * t; t = 0.5 / t;
    s.qw = (m02 - m20) * t; s.qz = (m21 + m12) * t; s.qx = (m01 + m10) * t;
  } else {
    double t = sqrt(m22 - m00 - m11 + 1.0);
    s.qz = 0.5 * t; t = 0.5 / t;
    s.qw = (m10 - m01) * t; s.qx = (m02 + m20) * t; s.qy = (m12 + m21) * t;
  }
  se3_normalize(s);
  s.tx = T[3]; s.ty = T[7]; s.tz = T[11];
  return s;
}

#define DVO_SE3_EPS 1e-10

// exp of a twist [vx vy vz wx wy wz]
DVO_HD SE3d se3_exp(const double a[6]) {
  const double wx = a[3], wy = a[4], wz = a[5];
  double theta = sqrt(wx * wx + wy * wy + wz * wz);
  double half = 0.5 * theta, imag, real;
  double sh = 0.0, ch = 1.0, st = 0.0, ct = 1.0;
  if (theta < DVO_SE3_EPS) {
    double t2 = theta * theta, t4 = t2 * t2;
    imag = 0.5 - t2 / 48.0 + t4 / 3840.0;
    real = 1.0 - t2 / 8.0 + t4 / 384.0;
  } else {
#ifdef __CUDA_ARCH__
    sincos(half, &sh, &ch);     // one argument reduction for the pair (same values as sin() / cos())
    sincos(theta, &st, &ct);
#else
    sh = sin(half); ch = cos(half); st = sin(theta); ct = cos(theta);
#endif
    imag = sh / theta;
    real = ch;
  }
  SE3d r;
  r.qw = real; r.qx = imag * wx; r.qy = imag * wy; r.qz = imag * wz;
  // V = I + c1*W + c2*W^2 ; applied to v without forming matrices: W v = w x v
  double c1, c2;
  if (theta < DVO_SE3_EPS) {
    // small angle: V ~= R (as the reference library does); R v = v + 2 qw (q x v) + 2 q x (q x v)
    double R[9];
    se3_rotation(r, R);
    r.tx = R[0] * a[0] + R[1] * a[1] + R[2] * a[2];
    r.ty = R[3] * a[0] + R[4] * a[1] + R[5] * a[2];
    r.tz = R[6] * a[0] + R[7] * a[1] + R[8] * a[2];
    return r;
  }
  double t2 = theta * theta;
  c1 = (1.0 - ct) / t2;
  c2 = (theta - st) / (t2 * theta);
  double cx = wy * a[2] - wz * a[1], cy = wz * a[0] - wx * a[2], cz = wx * a[1] - wy * a[0];  // w x v
  double dx = wy * cz - wz * cy, dy = wz * cx - wx * cz, dz = wx * cy - wy * cx;              // w x (w x v)
  r.tx = a[0] + c1 * cx + c2 * dx;
  r.ty = a[1] + c1 * cy + c2 * dy;
  r.tz = a[2] + c1 * cz + c2 * dz;
  return r;
}

DVO_HD void se3_log(const SE3d& s, double out[6]) {
  double sq = s.qx * s.qx + s.qy * s.qy + s.qz * s.qz;
  double n = sqrt(sq), w = s.qw, two_atan;
  if (n < DVO_SE3_EPS) {
    two_atan = 2.0 / w - 2.0 * sq / (w * w * w);
  } else if (fabs(w) < DVO_SE3_EPS) {
    two_atan = (w > 0 ? 3.14159265358979323846 : -3.14159265358979323846) / n;
  } else {
    two_atan = 2.0 * atan(n / w) / n;
  }
  double theta = two_atan * n;
  double wx = two_atan * s.qx, wy = two_atan * s.qy, wz = two_atan * s.qz;
  double c;
  if (fabs(theta) < DVO_SE3_EPS) {
    c = 1.0 / 12.0;
  } else {
    double half = 0.5 * theta;
    c = (1.0 - theta * cos(half) / (2.0 * sin(half))) / (theta * theta);
  }
  // V^-1 t = t - 0.5 w x t + c w x (w x t)
  double cx = wy * s.tz - wz * s.ty, cy = wz * s.tx - wx * s.tz, cz = wx * s.ty - wy * s.tx;
  double dx = wy * cz - wz * cy, dy = wz * cx - wx * cz, dz = wx * cy - wy * cx;
  out[0] = s.tx - 0.5 * cx + c * dx;
  out[1] = s.ty - 0.5 * cy + c * dy;
  out[2] = s.tz - 0.5 * cz + c * dz;
  out[3] = wx; out[4] = wy; out[5] = wz;
}

// x = A.ldlt().solve(b) for a symmetric 6x6 (diagonal pivoting, Eigen's tolerance rule on D).
//
// Eigen's unblocked LDL^T is left-looking: when step k searches the remaining diagonal for its pivot, the entries it
// compares have not been updated yet, so the whole pivot sequence is a selection sort of the ORIGINAL diagonal by
// decreasing magnitude (first maximum wins) and can be found up front.  Factorising the symmetrically permuted matrix
// without pivoting then performs exactly the operations of the in-place pivoted version, with compile-time indices:
// on the device everything stays in registers (the in-place version indexed a local-memory array through the
// permutation, ~700 local loads and stores on the critical path of every Gauss-Newton iteration).
// The same for any symmetric n x n (the 8 x 8 of the affine brightness model, tracker.cu).
template <int n>
DVO_HD void ldlt_solve(const double* Ain, const double* bin, double* x) {
  int idx[n];
#pragma unroll
  for (int i = 0; i < n; ++i) idx[i] = i;
#pragma unroll
  for (int k = 0; k < n; ++k) {
    int piv = k;
    double best = fabs(Ain[idx[k] * n + idx[k]]);
#pragma unroll
    for (int i = k + 1; i < n; ++i) {
      double v = fabs(Ain[idx[i] * n + idx[i]]);
      if (v > best) { best = v; piv = i; }
    }
    // swap idx[k] <-> idx[piv] with static indexing
    int ik = idx[k], ip = ik;
#pragma unroll
    for (int i = k + 1; i < n; ++i) if (piv == i) ip = idx[i];
#pragma unroll
    for (int i = k + 1; i < n; ++i) if (piv == i) idx[i] = ik;
    idx[k] = ip;
  }
  double A[n][n], y[n], rd[n];     // rd: reciprocal pivots (one division per pivot; Eigen divides element by element,
                                   // which differs in the last bit of a double -- far below every tolerance of this path)
#pragma unroll
  for (int i = 0; i < n; ++i) {
    y[i] = bin[idx[i]];
#pragma unroll
    for (int j = 0; j <= i; ++j) A[i][j] = Ain[idx[i] * n + idx[j]];     // lower triangle of P A P^T
  }
#pragma unroll
  for (int k = 0; k < n; ++k) {
#pragma unroll
    for (int j = 0; j < k; ++j) A[k][k] -= A[k][j] * A[k][j] * A[j][j];
    const double d = A[k][k];
    rd[k] = (d != 0.0) ? 1.0 / d : 0.0;
#pragma unroll
    for (int i = k + 1; i < n; ++i) {
      double s = A[i][k];
#pragma unroll
      for (int j = 0; j < k; ++j) s -= A[i][j] * A[k][j] * A[j][j];
      A[i][k] = s * rd[k];
    }
  }
#pragma unroll
  for (int i = 0; i < n; ++i)
#pragma unroll
    for (int j = 0; j < i; ++j) y[i] -= A[i][j] * y[j];
  double dmax = 0;
#pragma unroll
  for (int i = 0; i < n; ++i) dmax = fmax(dmax, fabs(A[i][i]));
  const double tol = fmax(dmax * DBL_EPSILON, 1.0 / DBL_MAX);
#pragma unroll
  for (int i = 0; i < n; ++i) y[i] = fabs(A[i][i]) > tol ? y[i] * rd[i] : 0.0;
#pragma unroll
  for (int i = n - 1; i >= 0; --i)
#pragma unroll
    for (int j = i + 1; j < n; ++j) y[i] -= A[j][i] * y[j];
#pragma unroll
  for (int i = 0; i < n; ++i) {
    // x[idx[i]] = y[i] with static indexing of x
#pragma unroll
    for (int t = 0; t < n; ++t) if (idx[i] == t) x[t] = y[i];
  }
}
DVO_HD void ldlt_solve6(const double Ain[36], const double bin[6], double x[6]) { ldlt_solve<6>(Ain, bin, x); }

}  // namespace dvo_b200
