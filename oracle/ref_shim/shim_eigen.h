// shim_eigen.h -- TEST INFRASTRUCTURE.  The smallest stand-in for the parts of Eigen 3 that the reference's SSE
// translation units touch, so that dvo_core/src/{dense_tracking_impl,core/math_sse,core/intrinsic_matrix}.cpp
// compile UNMODIFIED into oracle/_ref/ (Eigen itself is not in this image).  Those files use Eigen as a container
// (data(), operator(), fixed-size storage, column-major like Eigen's default) and for a handful of 2x2 / 3x4 expressions;
// the arithmetic that matters is their own SSE intrinsics.  Fixed-size products are plain loops in index order
// (a0*b0 + a1*b1 + ...), compiled with -ffp-contract=off.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstring>
#include <limits>
#include <memory>
#include <type_traits>
#include <vector>

#define EIGEN_ALIGN16 __attribute__((aligned(16)))
#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW

namespace Eigen {

enum { Dynamic = -1 };
enum { ColMajor = 0, RowMajor = 1 };
enum { Affine = 1 };
enum { Infinity = -1 };
enum { Upper = 2, Lower = 1 };
enum NoChange_t { NoChange };
enum { ComputeThinU = 1, ComputeThinV = 2, ComputeFullU = 4, ComputeFullV = 8 };

template <typename T> using aligned_allocator = std::allocator<T>;   // operator new is 16-byte aligned on x86-64

template <typename T, int R, int C, int Opt = ColMajor> class Matrix;

template <typename M> class CommaInit {
 public:
  CommaInit(M& m, typename M::Scalar v) : m_(m), i_(0) { put(v); }
  CommaInit& operator,(typename M::Scalar v) { put(v); return *this; }
 private:
  void put(typename M::Scalar v) { m_(i_ / M::Cols, i_ % M::Cols) = v; ++i_; }   // row by row, like Eigen
  M& m_; int i_;
};

// view of external memory as a fixed-size column-major matrix (Matrix::MapType / AlignedMapType / head<N>())
template <typename T, int R, int C> class Map {
 public:
  typedef typename std::remove_const<T>::type V;
  explicit Map(T* p) : p_(p) {}
  T& operator()(int i, int j) const { return p_[j * R + i]; }
  T& operator()(int i) const { return p_[i]; }
  T* data() const { return p_; }
  Matrix<V, R, C> eval() const { Matrix<V, R, C> m; for (int i = 0; i < R * C; ++i) m.data()[i] = p_[i]; return m; }
  operator Matrix<V, R, C>() const { return eval(); }
  const Map& operator=(const Matrix<V, R, C>& m) const { for (int i = 0; i < R * C; ++i) p_[i] = m.data()[i]; return *this; }
  const Map& operator=(const Map& o) const { for (int i = 0; i < R * C; ++i) p_[i] = o.p_[i]; return *this; }
 private:
  T* p_;
};

template <typename M> class SelfAdjointUpperView {
 public:
  explicit SelfAdjointUpperView(const M& m) : m_(m) {}
  void evalTo(M& out) const {
    for (int i = 0; i < M::Rows; ++i)
      for (int j = 0; j < M::Cols; ++j) out(i, j) = i <= j ? m_(i, j) : m_(j, i);
  }
 private:
  const M& m_;
};

template <typename T, int R, int C, int Opt>
class Matrix {
 public:
  typedef T Scalar;
  enum { Rows = R, Cols = C };
  typedef Map<T, R, C> MapType;
  typedef Map<T, R, C> AlignedMapType;
  typedef Map<const T, R, C> ConstMapType;
  typedef Map<const T, R, C> ConstAlignedMapType;

  Matrix() {}
  Matrix(T x, T y) { static_assert(R * C == 2, "size"); m_[0] = x; m_[1] = y; }
  Matrix(T x, T y, T z) { static_assert(R * C == 3, "size"); m_[0] = x; m_[1] = y; m_[2] = z; }
  Matrix(T x, T y, T z, T w) { static_assert(R * C == 4, "size"); m_[0] = x; m_[1] = y; m_[2] = z; m_[3] = w; }

  T& operator()(int i, int j) { return m_[j * R + i]; }
  const T& operator()(int i, int j) const { return m_[j * R + i]; }
  T& operator()(int i) { return m_[i]; }
  const T& operator()(int i) const { return m_[i]; }
  const T& coeff(int i) const { return m_[i]; }
  const T& coeff(int i, int j) const { return m_[j * R + i]; }
  T& operator[](int i) { return m_[i]; }
  const T& operator[](int i) const { return m_[i]; }
  T* data() { return m_; }
  const T* data() const { return m_; }
  operator T() const { static_assert(R == 1 && C == 1, "only a 1x1 expression converts to its scalar"); return m_[0]; }

  Matrix& setZero() { for (int i = 0; i < R * C; ++i) m_[i] = T(0); return *this; }
  Matrix& setConstant(T v) { for (int i = 0; i < R * C; ++i) m_[i] = v; return *this; }
  Matrix& setIdentity() { setZero(); for (int i = 0; i < (R < C ? R : C); ++i) (*this)(i, i) = T(1); return *this; }
  static Matrix Zero() { Matrix m; m.setZero(); return m; }
  static Matrix Identity() { Matrix m; m.setIdentity(); return m; }
  static Matrix Constant(T v) { Matrix m; m.setConstant(v); return m; }

  CommaInit<Matrix> operator<<(T v) { return CommaInit<Matrix>(*this, v); }

  Matrix<T, C, R> transpose() const {
    Matrix<T, C, R> t;
    for (int i = 0; i < R; ++i) for (int j = 0; j < C; ++j) t(j, i) = (*this)(i, j);
    return t;
  }
  template <int N> Map<T, N, 1> head() { static_assert(C == 1 && N <= R, "vector head"); return Map<T, N, 1>(m_); }
  Matrix cwiseProduct(const Matrix& o) const { Matrix r; for (int i = 0; i < R * C; ++i) r.m_[i] = m_[i] * o.m_[i]; return r; }
  template <int BR, int BC> Matrix<T, BR, BC> block(int i0, int j0) const {
    Matrix<T, BR, BC> b;
    for (int i = 0; i < BR; ++i) for (int j = 0; j < BC; ++j) b(i, j) = (*this)(i0 + i, j0 + j);
    return b;
  }
  template <typename U> Matrix<U, R, C> cast() const {
    Matrix<U, R, C> o;
    for (int i = 0; i < R * C; ++i) o.data()[i] = (U)m_[i];
    return o;
  }
  T sum() const { T a = m_[0]; for (int i = 1; i < R * C; ++i) a += m_[i]; return a; }
  T squaredNorm() const { T a = m_[0] * m_[0]; for (int i = 1; i < R * C; ++i) a += m_[i] * m_[i]; return a; }
  T determinant() const {
    static_assert(R == C, "square only");
    if (R == 2) return m_[0] * m_[3] - m_[2] * m_[1];
    T a[R * C];   // partial-pivot LU (only the 2x2 closed form is used by the reference's translation units)
    for (int i = 0; i < R * C; ++i) a[i] = m_[i];
    T det = T(1);
    for (int k = 0; k < R; ++k) {
      int piv = k;
      for (int i = k + 1; i < R; ++i) if (std::fabs(a[k * R + i]) > std::fabs(a[k * R + piv])) piv = i;
      if (a[k * R + piv] == T(0)) return T(0);
      if (piv != k) { for (int j = 0; j < C; ++j) { T t = a[j * R + k]; a[j * R + k] = a[j * R + piv]; a[j * R + piv] = t; } det = -det; }
      det *= a[k * R + k];
      for (int i = k + 1; i < R; ++i) {
        const T f = a[k * R + i] / a[k * R + k];
        for (int j = k; j < C; ++j) a[j * R + i] -= f * a[j * R + k];
      }
    }
    return det;
  }
  Matrix inverse() const {   // Eigen's 2x2 inverse: adjugate times 1/det
    static_assert(R == 2 && C == 2, "2x2 only");
    const T invdet = T(1) / determinant();
    Matrix r;
    r(0, 0) = (*this)(1, 1) * invdet; r(1, 0) = -(*this)(1, 0) * invdet;
    r(0, 1) = -(*this)(0, 1) * invdet; r(1, 1) = (*this)(0, 0) * invdet;
    return r;
  }
  template <int P> T lpNorm() const {
    static_assert(P == Infinity, "only the infinity norm");
    T m = T(0);
    for (int i = 0; i < R * C; ++i) m = std::fabs(m_[i]) > m ? std::fabs(m_[i]) : m;
    return m;
  }
  template <int UpLo> SelfAdjointUpperView<Matrix> selfadjointView() const {
    static_assert(UpLo == Upper, "upper only");
    return SelfAdjointUpperView<Matrix>(*this);
  }

  Matrix operator-() const { Matrix r; for (int i = 0; i < R * C; ++i) r.m_[i] = -m_[i]; return r; }
  Matrix& operator+=(const Matrix& o) { for (int i = 0; i < R * C; ++i) m_[i] += o.m_[i]; return *this; }
  Matrix& operator-=(const Matrix& o) { for (int i = 0; i < R * C; ++i) m_[i] -= o.m_[i]; return *this; }
  Matrix& operator*=(T s) { for (int i = 0; i < R * C; ++i) m_[i] *= s; return *this; }
  Matrix& operator/=(T s) { for (int i = 0; i < R * C; ++i) m_[i] /= s; return *this; }

 private:
  // Eigen aligns fixed-size objects to 16 bytes exactly when their size is a multiple of 16 bytes (Vector4f, Matrix2f,
  // Matrix<float,2,6>, ...); Vector2f stays 8 bytes, which the SSE loops rely on (two residuals per 128-bit load)
  alignas((sizeof(T) * R * C) % 16 == 0 ? 16 : alignof(T)) T m_[R * C];
};

// dynamic sizes only occur in member declarations of classes these translation units never instantiate
template <typename T, int C, int Opt> class Matrix<T, Dynamic, C, Opt> { std::vector<T> v_; };
template <typename T, int R, int Opt> class Matrix<T, R, Dynamic, Opt> { std::vector<T> v_; };

template <typename T, int R, int C> Matrix<T, R, C> operator+(const Matrix<T, R, C>& a, const Matrix<T, R, C>& b) { Matrix<T, R, C> r = a; r += b; return r; }
template <typename T, int R, int C> Matrix<T, R, C> operator-(const Matrix<T, R, C>& a, const Matrix<T, R, C>& b) { Matrix<T, R, C> r = a; r -= b; return r; }
template <typename T, int R, int C> Matrix<T, R, C> operator*(const Matrix<T, R, C>& a, T s) { Matrix<T, R, C> r = a; r *= s; return r; }
template <typename T, int R, int C> Matrix<T, R, C> operator*(T s, const Matrix<T, R, C>& a) { Matrix<T, R, C> r = a; r *= s; return r; }
template <typename T, int R, int C> Matrix<T, R, C> operator/(const Matrix<T, R, C>& a, T s) { Matrix<T, R, C> r = a; r /= s; return r; }
template <typename T, int R, int K, int C>
Matrix<T, R, C> operator*(const Matrix<T, R, K>& a, const Matrix<T, K, C>& b) {
  Matrix<T, R, C> r;
  for (int i = 0; i < R; ++i)
    for (int j = 0; j < C; ++j) {
      T acc = a(i, 0) * b(0, j);
      for (int k = 1; k < K; ++k) acc += a(i, k) * b(k, j);
      r(i, j) = acc;
    }
  return r;
}

// expressions on maps evaluate the map first
template <typename T, int R, int C> Matrix<typename Map<T, R, C>::V, R, C> operator*(const Map<T, R, C>& a, typename Map<T, R, C>::V s) { return a.eval() * s; }
template <typename T, typename T2, int R, int K, int C>
Matrix<T, R, C> operator*(const Matrix<T, R, K>& a, const Map<T2, K, C>& b) { return a * b.eval(); }

template <typename T, int Dim, int Mode>
class Transform {
 public:
  typedef Matrix<T, Dim + 1, Dim + 1> MatrixType;
  Transform() {}
  MatrixType& matrix() { return m_; }
  const MatrixType& matrix() const { return m_; }
  void setIdentity() { m_.setIdentity(); }
  T& operator()(int i, int j) { return m_(i, j); }
  const T& operator()(int i, int j) const { return m_(i, j); }
  static Transform Identity() { Transform t; t.setIdentity(); return t; }
  Matrix<T, Dim, Dim> rotation() const { return m_.template block<Dim, Dim>(0, 0); }
  Matrix<T, Dim, Dim> linear() const { return rotation(); }
  Matrix<T, Dim, 1> translation() const { return m_.template block<Dim, 1>(0, Dim); }
  Transform operator*(const Transform& o) const { Transform r; r.m_ = m_ * o.m_; return r; }
  Transform inverse() const {   // rigid-body inverse (Affine mode with an orthonormal linear part)
    Transform r; r.setIdentity();
    for (int i = 0; i < Dim; ++i) for (int j = 0; j < Dim; ++j) r.m_(i, j) = m_(j, i);
    for (int i = 0; i < Dim; ++i) { T s = T(0); for (int k = 0; k < Dim; ++k) s += m_(k, i) * m_(k, Dim); r.m_(i, Dim) = -s; }
    return r;
  }
  template <typename U> Transform<U, Dim, Mode> cast() const { Transform<U, Dim, Mode> t; t.matrix() = m_.template cast<U>(); return t; }
 private:
  MatrixType m_;
};

typedef Matrix<float, 2, 2> Matrix2f;  typedef Matrix<double, 2, 2> Matrix2d;
typedef Matrix<float, 3, 3> Matrix3f;  typedef Matrix<double, 3, 3> Matrix3d;
typedef Matrix<float, 4, 4> Matrix4f;  typedef Matrix<double, 4, 4> Matrix4d;
typedef Matrix<float, 2, 1> Vector2f;  typedef Matrix<double, 2, 1> Vector2d;
typedef Matrix<float, 3, 1> Vector3f;  typedef Matrix<double, 3, 1> Vector3d;
typedef Matrix<float, 4, 1> Vector4f;  typedef Matrix<double, 4, 1> Vector4d;
typedef Transform<float, 3, Affine> Affine3f;
typedef Transform<double, 3, Affine> Affine3d;

}  // namespace Eigen
