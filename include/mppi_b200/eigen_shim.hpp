/*
 * mppi_b200/eigen_shim.hpp — the few fixed-size, column-major matrix facilities the host layer needs, used ONLY when
 * Eigen itself is not installed (this image has no Eigen; SURVEY.md §0). With Eigen present the host layer includes
 * <Eigen/Dense> and this file is skipped, so user code written against the reference (Eigen::Matrix, Eigen::Ref,
 * .col(), .block(), Zero(), comma initialiser) compiles unchanged either way.
 *
 * Scope: float matrices with compile-time sizes, column-major storage (so a C x T control_trajectory is the engine's
 * [t][c] layout), element access, col()/block() views, Zero/Ones/Constant/setZero, +,-,scalar *, ==, <<.
 */
#pragma once
#if defined(MPPIB_FORCE_EIGEN_SHIM) || !__has_include(<Eigen/Dense>)
#define MPPIB_USING_EIGEN_SHIM 1
#include <cassert>
#include <cstring>
#include <iostream>
#include <type_traits>

namespace Eigen
{
template <class Derived>
struct DenseBase
{
};

// strided view on float storage (column-major with leading dimension ld)
template <bool Const>
class View : public DenseBase<View<Const>>
{
public:
  using ptr_t = typename std::conditional<Const, const float*, float*>::type;
  View(ptr_t p, int r, int c, int ld) : p_(p), r_(r), c_(c), ld_(ld)
  {
  }
  int rows() const
  {
    return r_;
  }
  int cols() const
  {
    return c_;
  }
  int size() const
  {
    return r_ * c_;
  }
  float operator()(int i, int j) const
  {
    return p_[i + (long)j * ld_];
  }
  float operator()(int i) const
  {
    return (c_ == 1) ? p_[i] : p_[(long)i * ld_];
  }
  float operator[](int i) const
  {
    return (*this)(i);
  }
  template <bool C2 = Const, typename std::enable_if<!C2, int>::type = 0>
  float& operator()(int i, int j)
  {
    return p_[i + (long)j * ld_];
  }
  template <bool C2 = Const, typename std::enable_if<!C2, int>::type = 0>
  float& operator()(int i)
  {
    return (c_ == 1) ? p_[i] : p_[(long)i * ld_];
  }
  template <bool C2 = Const, typename std::enable_if<!C2, int>::type = 0>
  float& operator[](int i)
  {
    return (*this)(i);
  }
  ptr_t data() const
  {
    return p_;
  }
  int outerStride() const
  {
    return ld_;
  }
  // assignment copies element-wise (views never rebind)
  template <class Other, bool C2 = Const, typename std::enable_if<!C2, int>::type = 0>
  View& operator=(const DenseBase<Other>& o_)
  {
    const Other& o = static_cast<const Other&>(o_);
    assert(o.rows() == r_ && o.cols() == c_);
    for (int j = 0; j < c_; j++)
      for (int i = 0; i < r_; i++)
        (*this)(i, j) = o(i, j);
    return *this;
  }
  template <bool C2 = Const, typename std::enable_if<!C2, int>::type = 0>
  View& operator=(const View& o)
  {
    for (int j = 0; j < c_; j++)
      for (int i = 0; i < r_; i++)
        (*this)(i, j) = o(i, j);
    return *this;
  }
  View<Const> col(int j) const
  {
    return View<Const>(p_ + (long)j * ld_, r_, 1, ld_);
  }
  View<Const> block(int i, int j, int nr, int nc) const
  {
    return View<Const>(p_ + i + (long)j * ld_, nr, nc, ld_);
  }

private:
  ptr_t p_;
  int r_, c_, ld_;
};

template <class T, int R, int C, int = 0, int = R, int = C>
class Matrix : public DenseBase<Matrix<T, R, C>>
{
  static_assert(std::is_same<T, float>::value, "eigen_shim only provides float matrices");
  static_assert(R > 0 && C > 0, "eigen_shim only provides fixed-size matrices");

public:
  enum
  {
    RowsAtCompileTime = R,
    ColsAtCompileTime = C,
    SizeAtCompileTime = R * C
  };
  Matrix()
  {
  }
  template <class Other>
  Matrix(const DenseBase<Other>& o_)
  {
    *this = o_;
  }
  template <class Other>
  Matrix& operator=(const DenseBase<Other>& o_)
  {
    const Other& o = static_cast<const Other&>(o_);
    assert(o.rows() == R && o.cols() == C);
    for (int j = 0; j < C; j++)
      for (int i = 0; i < R; i++)
        d_[i + j * R] = o(i, j);
    return *this;
  }
  static Matrix Zero()
  {
    return Constant(0.0f);
  }
  static Matrix Ones()
  {
    return Constant(1.0f);
  }
  static Matrix Constant(float v)
  {
    Matrix m;
    for (int i = 0; i < R * C; i++)
      m.d_[i] = v;
    return m;
  }
  static Matrix Identity()
  {
    Matrix m = Zero();
    for (int i = 0; i < R && i < C; i++)
      m.d_[i + i * R] = 1.0f;
    return m;
  }
  void setIdentity()
  {
    *this = Identity();
  }
  void setZero()
  {
    memset(d_, 0, sizeof(d_));
  }
  void setConstant(float v)
  {
    for (int i = 0; i < R * C; i++)
      d_[i] = v;
  }
  int rows() const
  {
    return R;
  }
  int cols() const
  {
    return C;
  }
  int size() const
  {
    return R * C;
  }
  float* data()
  {
    return d_;
  }
  const float* data() const
  {
    return d_;
  }
  float& operator()(int i, int j)
  {
    return d_[i + j * R];
  }
  float operator()(int i, int j) const
  {
    return d_[i + j * R];
  }
  float& operator()(int i)
  {
    return d_[i];
  }
  float operator()(int i) const
  {
    return d_[i];
  }
  float& operator[](int i)
  {
    return d_[i];
  }
  float operator[](int i) const
  {
    return d_[i];
  }
  View<false> col(int j)
  {
    return View<false>(d_ + j * R, R, 1, R);
  }
  View<true> col(int j) const
  {
    return View<true>(d_ + j * R, R, 1, R);
  }
  View<false> block(int i, int j, int nr, int nc)
  {
    return View<false>(d_ + i + j * R, nr, nc, R);
  }
  View<true> block(int i, int j, int nr, int nc) const
  {
    return View<true>(d_ + i + j * R, nr, nc, R);
  }
  Matrix operator+(const Matrix& o) const
  {
    Matrix m;
    for (int i = 0; i < R * C; i++)
      m.d_[i] = d_[i] + o.d_[i];
    return m;
  }
  Matrix operator-(const Matrix& o) const
  {
    Matrix m;
    for (int i = 0; i < R * C; i++)
      m.d_[i] = d_[i] - o.d_[i];
    return m;
  }
  Matrix operator*(float s) const
  {
    Matrix m;
    for (int i = 0; i < R * C; i++)
      m.d_[i] = d_[i] * s;
    return m;
  }
  Matrix& operator+=(const Matrix& o)
  {
    for (int i = 0; i < R * C; i++)
      d_[i] += o.d_[i];
    return *this;
  }
  bool operator==(const Matrix& o) const
  {
    return memcmp(d_, o.d_, sizeof(d_)) == 0;
  }
  // comma initialiser: m << a, b, c;  (row-major order, like Eigen)
  struct CommaInit
  {
    Matrix& m;
    int k;
    CommaInit& operator,(float v)
    {
      assert(k < R * C);
      m.d_[(k / C) + (k % C) * R] = v;
      k++;
      return *this;
    }
  };
  CommaInit operator<<(float v)
  {
    d_[0] = v;
    return CommaInit{ *this, 1 };
  }
  // m.diagonal() << a, b, c;  (the reference's examples set DDP weights this way)
  struct DiagonalInit
  {
    Matrix& m;
    int k;
    DiagonalInit& operator,(float v)
    {
      assert(k < (R < C ? R : C));
      m.d_[k + k * R] = v;
      k++;
      return *this;
    }
  };
  struct Diagonal
  {
    Matrix& m;
    DiagonalInit operator<<(float v)
    {
      m.d_[0] = v;
      return DiagonalInit{ m, 1 };
    }
    float operator()(int i) const
    {
      return m.d_[i + i * R];
    }
  };
  Diagonal diagonal()
  {
    return Diagonal{ *this };
  }

private:
  float d_[R * C];
};

template <class T, int R, int C>
inline Matrix<T, R, C> operator*(float s, const Matrix<T, R, C>& m)
{
  return m * s;
}
template <class T, int R, int C>
inline std::ostream& operator<<(std::ostream& os, const Matrix<T, R, C>& m)
{
  for (int i = 0; i < R; i++)
  {
    for (int j = 0; j < C; j++)
      os << m(i, j) << (j + 1 < C ? " " : "");
    os << (i + 1 < R ? "\n" : "");
  }
  return os;
}

// Eigen::Ref<const M> / Eigen::Ref<M>: non-owning argument types. Constructible from a Matrix of the same shape or
// from a column / block view.
template <class M>
class Ref;
template <class T, int R, int C>
class Ref<const Matrix<T, R, C>> : public View<true>
{
public:
  Ref(const Matrix<T, R, C>& m) : View<true>(m.data(), R, C, R)
  {
  }
  template <bool Cn>
  Ref(const View<Cn>& v) : View<true>(v.data(), v.rows(), v.cols(), v.outerStride())
  {
    assert(v.rows() == R && v.cols() == C);
  }
};
template <class T, int R, int C>
class Ref<Matrix<T, R, C>> : public View<false>
{
public:
  Ref(Matrix<T, R, C>& m) : View<false>(m.data(), R, C, R)
  {
  }
  Ref(const View<false>& v) : View<false>(v.data(), v.rows(), v.cols(), v.outerStride())
  {
    assert(v.rows() == R && v.cols() == C);
  }
  using View<false>::operator=;
};

typedef Matrix<float, 3, 3> Matrix3f;
typedef Matrix<float, 3, 1> Vector3f;

// unit quaternion (w, x, y, z) with the accessors, conjugate, rotation matrix and vector rotation the host layer uses
class Quaternionf
{
public:
  Quaternionf() : w_(1.0f), x_(0.0f), y_(0.0f), z_(0.0f)
  {
  }
  Quaternionf(float w, float x, float y, float z) : w_(w), x_(x), y_(y), z_(z)
  {
  }
  float w() const
  {
    return w_;
  }
  float x() const
  {
    return x_;
  }
  float y() const
  {
    return y_;
  }
  float z() const
  {
    return z_;
  }
  Quaternionf conjugate() const
  {
    return Quaternionf(w_, -x_, -y_, -z_);
  }
  Matrix3f toRotationMatrix() const
  {  // Eigen's formula
    const float tx = 2 * x_, ty = 2 * y_, tz = 2 * z_, twx = tx * w_, twy = ty * w_, twz = tz * w_, txx = tx * x_,
                txy = ty * x_, txz = tz * x_, tyy = ty * y_, tyz = tz * y_, tzz = tz * z_;
    Matrix3f m;
    m << 1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx,
        1 - (txx + tyy);
    return m;
  }
  Vector3f operator*(const Vector3f& v) const
  {
    const Matrix3f m = toRotationMatrix();
    Vector3f r;
    for (int i = 0; i < 3; i++)
      r(i) = m(i, 0) * v(0) + m(i, 1) * v(1) + m(i, 2) * v(2);
    return r;
  }

private:
  float w_, x_, y_, z_;
};
}  // namespace Eigen
#else
#include <Eigen/Dense>
#endif
