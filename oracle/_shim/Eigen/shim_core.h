// shim_core.h -- a small eager-evaluation stand-in for the parts of Eigen 3 that the D2SLAM factor sources use.
//
// TEST INFRASTRUCTURE ONLY (oracle/_ref build).  Eigen is not installed in this image, so the reference's factor
// sources (d2vins/src/factors/*.cpp, d2common/src/solver/consenus_factor.cpp, ...) are compiled UNMODIFIED against
// this header set.  It is NOT a copy of Eigen: there are no expression templates, every operation returns a plain
// Matrix.  The arithmetic that matters for parity (products, sums, quaternion rotation, toRotationMatrix) follows the
// formulas Eigen documents, evaluated in the same order for the small fixed sizes used here.
#pragma once
#include <algorithm>
#include <cassert>
#include <cmath>
#include <complex>
#include <iostream>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

namespace Eigen {
constexpr int Dynamic = -1;
enum { ColMajor = 0, RowMajor = 1, AutoAlign = 0, DontAlign = 2 };
enum { ComputeFullU = 4, ComputeThinU = 8, ComputeFullV = 16, ComputeThinV = 32 };
enum ComputationInfo { Success = 0, NumericalIssue = 1, NoConvergence = 2, InvalidInput = 3 };
enum { StreamPrecision = -1, FullPrecision = -2 };
enum { DontAlignCols = 1 };
typedef std::ptrdiff_t Index;

struct IOFormat {
  IOFormat(int = StreamPrecision, int = 0, const std::string & = " ", const std::string & = "\n", const std::string & = "",
           const std::string & = "", const std::string & = "", const std::string & = "") {}
};

template <class Derived> struct traits;
template <class S, int R, int C, int Opt = 0, int MR = R, int MC = C> class Matrix;
template <class X, int BR, int BC> class Block;
template <class M, int MapOpt = 0, class Stride = void> class Map;
template <class S, int Opt = 0> class Quaternion;
template <class Derived> class QuaternionBase;
template <class M> class JacobiSVD;

template <class T> struct traits<const T> : traits<T> {};
template <class S, int R, int C, int Opt, int MR, int MC> struct traits<Matrix<S, R, C, Opt, MR, MC>> {
  typedef S Scalar;
  enum { Rows = R, Cols = C, Options = Opt };
};
template <class X, int BR, int BC> struct traits<Block<X, BR, BC>> {
  typedef typename traits<X>::Scalar Scalar;
  enum { Rows = BR, Cols = BC, Options = 0 };
};
template <class M, int MO, class St> struct traits<Map<M, MO, St>> : traits<M> {};

namespace shim {
constexpr int pick(int a, int b) { return a != Dynamic ? a : b; }
template <class S> struct CommaInit;
}  // namespace shim

// ------------------------------------------------------------------------------------------------ MatrixBase
template <class Derived>
class MatrixBase {
 public:
  typedef typename traits<Derived>::Scalar Scalar;
  enum { RowsAtCompileTime = traits<Derived>::Rows, ColsAtCompileTime = traits<Derived>::Cols,
         IsVectorAtCompileTime = (traits<Derived>::Rows == 1 || traits<Derived>::Cols == 1) };
  typedef Matrix<Scalar, RowsAtCompileTime, ColsAtCompileTime> PlainObject;
  typedef Matrix<Scalar, ColsAtCompileTime, RowsAtCompileTime> TransposeReturn;

  Derived &derived() { return *static_cast<Derived *>(this); }
  const Derived &derived() const { return *static_cast<const Derived *>(this); }
  int rows() const { return derived().rows_(); }
  int cols() const { return derived().cols_(); }
  int size() const { return rows() * cols(); }
  Scalar coeff(int i, int j) const { return derived().get(i, j); }
  Scalar &coeffRef(int i, int j) { return derived().ref(i, j); }
  Scalar operator()(int i, int j) const { return coeff(i, j); }
  Scalar &operator()(int i, int j) { return coeffRef(i, j); }
  // vector access
  Scalar vget(int i) const { return cols() == 1 ? coeff(i, 0) : coeff(0, i); }
  Scalar &vref(int i) { return cols() == 1 ? coeffRef(i, 0) : coeffRef(0, i); }
  Scalar operator()(int i) const { return vget(i); }
  Scalar &operator()(int i) { return vref(i); }
  Scalar operator[](int i) const { return vget(i); }
  Scalar &operator[](int i) { return vref(i); }
  Scalar x() const { return vget(0); }
  Scalar y() const { return vget(1); }
  Scalar z() const { return vget(2); }
  Scalar w() const { return vget(3); }
  Scalar &x() { return vref(0); }
  Scalar &y() { return vref(1); }
  Scalar &z() { return vref(2); }
  Scalar &w() { return vref(3); }

  PlainObject eval() const { return PlainObject(*this); }
  template <class T> Matrix<T, RowsAtCompileTime, ColsAtCompileTime> cast() const {
    Matrix<T, RowsAtCompileTime, ColsAtCompileTime> r(rows(), cols());
    for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) r.ref(i, j) = T(coeff(i, j));
    return r;
  }
  TransposeReturn transpose() const {
    TransposeReturn t(cols(), rows());
    for (int i = 0; i < rows(); i++) for (int j = 0; j < cols(); j++) t.ref(j, i) = coeff(i, j);
    return t;
  }
  Scalar squaredNorm() const { Scalar s = 0; for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) s += coeff(i, j) * coeff(i, j); return s; }
  Scalar norm() const { using std::sqrt; return sqrt(squaredNorm()); }
  PlainObject normalized() const { PlainObject r(*this); Scalar n2 = squaredNorm(); if (n2 > Scalar(0)) { using std::sqrt; Scalar n = sqrt(n2); for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) r.ref(i, j) = coeff(i, j) / n; } return r; }
  void normalize() { PlainObject r = normalized(); assign(r); }
  template <class O> Scalar dot(const MatrixBase<O> &o) const { Scalar s = 0; for (int i = 0; i < size(); i++) s += vget(i) * o.vget(i); return s; }
  template <class O> Matrix<Scalar, 3, 1> cross(const MatrixBase<O> &o) const {
    Matrix<Scalar, 3, 1> r;
    r(0) = vget(1) * o.vget(2) - vget(2) * o.vget(1);
    r(1) = vget(2) * o.vget(0) - vget(0) * o.vget(2);
    r(2) = vget(0) * o.vget(1) - vget(1) * o.vget(0);
    return r;
  }
  Scalar sum() const { Scalar s = 0; for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) s += coeff(i, j); return s; }
  Scalar trace() const { Scalar s = 0; for (int i = 0; i < rows(); i++) s += coeff(i, i); return s; }
  Scalar maxCoeff() const { Scalar m = coeff(0, 0); for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) m = std::max(m, coeff(i, j)); return m; }
  Scalar minCoeff() const { Scalar m = coeff(0, 0); for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) m = std::min(m, coeff(i, j)); return m; }
  bool hasNaN() const { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) if (coeff(i, j) != coeff(i, j)) return true; return false; }
  bool allFinite() const { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) if (!std::isfinite(coeff(i, j))) return false; return true; }
  PlainObject cwiseAbs() const { PlainObject r(*this); for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) r.ref(i, j) = std::fabs(coeff(i, j)); return r; }
  Scalar determinant() const;
  PlainObject inverse() const;
  JacobiSVD<PlainObject> jacobiSvd(int opts = 0) const;
  const Derived &format(const IOFormat &) const { return derived(); }

  // ---- assignment helpers
  template <class O> void assign(const MatrixBase<O> &o) {
    derived().resize_(o.rows(), o.cols());
    assert(rows() == o.rows() && cols() == o.cols());
    for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) = o.coeff(i, j);
  }
  template <class O> Derived &operator+=(const MatrixBase<O> &o) { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) += o.coeff(i, j); return derived(); }
  template <class O> Derived &operator-=(const MatrixBase<O> &o) { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) -= o.coeff(i, j); return derived(); }
  Derived &operator*=(const Scalar &s) { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) *= s; return derived(); }
  Derived &operator/=(const Scalar &s) { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) /= s; return derived(); }
  Derived &setZero() { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) = Scalar(0); return derived(); }
  Derived &setConstant(const Scalar &v) { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) = v; return derived(); }
  Derived &setIdentity() { for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) coeffRef(i, j) = i == j ? Scalar(1) : Scalar(0); return derived(); }
  template <class O> void applyOnTheLeft(const MatrixBase<O> &m);
  template <class O> void applyOnTheRight(const MatrixBase<O> &m);
  shim::CommaInit<Derived> operator<<(const Scalar &v);

  // ---- blocks
  template <int BR, int BC> Block<Derived, BR, BC> block(int i, int j) { return Block<Derived, BR, BC>(derived(), i, j, BR, BC); }
  template <int BR, int BC> Block<const Derived, BR, BC> block(int i, int j) const { return Block<const Derived, BR, BC>(derived(), i, j, BR, BC); }
  Block<Derived, Dynamic, Dynamic> block(int i, int j, int r, int c) { return Block<Derived, Dynamic, Dynamic>(derived(), i, j, r, c); }
  Block<const Derived, Dynamic, Dynamic> block(int i, int j, int r, int c) const { return Block<const Derived, Dynamic, Dynamic>(derived(), i, j, r, c); }
#define SHIM_FIXED_BLOCK(NAME, TPARAMS, BR, BC, I, J)                                                                        \
  template <TPARAMS> Block<Derived, BR, BC> NAME() { return Block<Derived, BR, BC>(derived(), I, J, pickdim(BR, rows()), pickdim(BC, cols())); }       \
  template <TPARAMS> Block<const Derived, BR, BC> NAME() const { return Block<const Derived, BR, BC>(derived(), I, J, pickdim(BR, rows()), pickdim(BC, cols())); }
  static constexpr int pickdim(int fixed, int dyn) { return fixed != Dynamic ? fixed : dyn; }
  SHIM_FIXED_BLOCK(leftCols, int N, RowsAtCompileTime, N, 0, 0)
  SHIM_FIXED_BLOCK(rightCols, int N, RowsAtCompileTime, N, 0, cols() - N)
  SHIM_FIXED_BLOCK(topRows, int N, N, ColsAtCompileTime, 0, 0)
  SHIM_FIXED_BLOCK(bottomRows, int N, N, ColsAtCompileTime, rows() - N, 0)
#undef SHIM_FIXED_BLOCK
  template <int BR, int BC> Block<Derived, BR, BC> topLeftCorner() { return block<BR, BC>(0, 0); }
  template <int BR, int BC> Block<const Derived, BR, BC> topLeftCorner() const { return block<BR, BC>(0, 0); }
  template <int BR, int BC> Block<Derived, BR, BC> bottomRightCorner() { return block<BR, BC>(rows() - BR, cols() - BC); }
  template <int BR, int BC> Block<const Derived, BR, BC> bottomRightCorner() const { return block<BR, BC>(rows() - BR, cols() - BC); }
  template <int BR, int BC> Block<Derived, BR, BC> topRightCorner() { return block<BR, BC>(0, cols() - BC); }
  template <int BR, int BC> Block<const Derived, BR, BC> topRightCorner() const { return block<BR, BC>(0, cols() - BC); }
  template <int BR, int BC> Block<Derived, BR, BC> bottomLeftCorner() { return block<BR, BC>(rows() - BR, 0); }
  template <int BR, int BC> Block<const Derived, BR, BC> bottomLeftCorner() const { return block<BR, BC>(rows() - BR, 0); }
  Block<Derived, Dynamic, Dynamic> leftCols(int n) { return block(0, 0, rows(), n); }
  Block<const Derived, Dynamic, Dynamic> leftCols(int n) const { return block(0, 0, rows(), n); }
  Block<Derived, Dynamic, Dynamic> middleCols(int j, int n) { return block(0, j, rows(), n); }
  Block<const Derived, Dynamic, Dynamic> middleCols(int j, int n) const { return block(0, j, rows(), n); }
  Block<Derived, Dynamic, Dynamic> middleRows(int i, int n) { return block(i, 0, n, cols()); }
  Block<const Derived, Dynamic, Dynamic> middleRows(int i, int n) const { return block(i, 0, n, cols()); }
  Block<Derived, Dynamic, Dynamic> rightCols(int n) { return block(0, cols() - n, rows(), n); }
  Block<const Derived, Dynamic, Dynamic> rightCols(int n) const { return block(0, cols() - n, rows(), n); }
  Block<Derived, Dynamic, Dynamic> topRows(int n) { return block(0, 0, n, cols()); }
  Block<const Derived, Dynamic, Dynamic> topRows(int n) const { return block(0, 0, n, cols()); }
  Block<Derived, Dynamic, Dynamic> bottomRows(int n) { return block(rows() - n, 0, n, cols()); }
  Block<const Derived, Dynamic, Dynamic> bottomRows(int n) const { return block(rows() - n, 0, n, cols()); }
  Block<Derived, RowsAtCompileTime, 1> col(int j) { return Block<Derived, RowsAtCompileTime, 1>(derived(), 0, j, rows(), 1); }
  Block<const Derived, RowsAtCompileTime, 1> col(int j) const { return Block<const Derived, RowsAtCompileTime, 1>(derived(), 0, j, rows(), 1); }
  Block<Derived, 1, ColsAtCompileTime> row(int i) { return Block<Derived, 1, ColsAtCompileTime>(derived(), i, 0, 1, cols()); }
  Block<const Derived, 1, ColsAtCompileTime> row(int i) const { return Block<const Derived, 1, ColsAtCompileTime>(derived(), i, 0, 1, cols()); }
  // vector segments (column or row vectors)
  template <int N> struct Seg { typedef Block<Derived, (ColsAtCompileTime == 1 ? N : 1), (ColsAtCompileTime == 1 ? 1 : N)> type;
                                typedef Block<const Derived, (ColsAtCompileTime == 1 ? N : 1), (ColsAtCompileTime == 1 ? 1 : N)> ctype; };
  template <int N> typename Seg<N>::type segment(int i) { return cols() == 1 ? typename Seg<N>::type(derived(), i, 0, N, 1) : typename Seg<N>::type(derived(), 0, i, 1, N); }
  template <int N> typename Seg<N>::ctype segment(int i) const { return cols() == 1 ? typename Seg<N>::ctype(derived(), i, 0, N, 1) : typename Seg<N>::ctype(derived(), 0, i, 1, N); }
  template <int N> typename Seg<N>::type head() { return segment<N>(0); }
  template <int N> typename Seg<N>::ctype head() const { return segment<N>(0); }
  template <int N> typename Seg<N>::type tail() { return segment<N>(size() - N); }
  template <int N> typename Seg<N>::ctype tail() const { return segment<N>(size() - N); }
  Block<Derived, Dynamic, Dynamic> segment(int i, int n) { return cols() == 1 ? block(i, 0, n, 1) : block(0, i, 1, n); }
  Block<const Derived, Dynamic, Dynamic> segment(int i, int n) const { return cols() == 1 ? block(i, 0, n, 1) : block(0, i, 1, n); }
  Block<Derived, Dynamic, Dynamic> head(int n) { return segment(0, n); }
  Block<const Derived, Dynamic, Dynamic> head(int n) const { return segment(0, n); }
  Block<Derived, Dynamic, Dynamic> tail(int n) { return segment(size() - n, n); }
  Block<const Derived, Dynamic, Dynamic> tail(int n) const { return segment(size() - n, n); }
  // coefficient-wise helpers (eager); array() supports the `(a.array() > eps).select(a.array()[.inverse()], 0)` idiom
  PlainObject cwiseSqrt() const { PlainObject r(*this); for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) { using std::sqrt; r.ref(i, j) = sqrt(coeff(i, j)); } return r; }
  PlainObject cwiseInverse() const { PlainObject r(*this); for (int j = 0; j < cols(); j++) for (int i = 0; i < rows(); i++) r.ref(i, j) = Scalar(1) / coeff(i, j); return r; }
  struct ArrayMask;
  struct ArrayView {
    PlainObject m;
    ArrayView inverse() const { ArrayView r{m.cwiseInverse()}; return r; }
    ArrayView sqrt() const { ArrayView r{m.cwiseSqrt()}; return r; }
    ArrayMask operator>(const Scalar &t) const { ArrayMask k; k.rows = m.rows(); k.cols = m.cols(); k.b.resize((size_t)m.rows() * m.cols()); for (int j = 0; j < m.cols(); j++) for (int i = 0; i < m.rows(); i++) k.b[(size_t)j * m.rows() + i] = m.coeff(i, j) > t; return k; }
    operator PlainObject() const { return m; }
    PlainObject matrix() const { return m; }
  };
  struct ArrayMask {
    std::vector<char> b; int rows = 0, cols = 0;
    PlainObject select(const ArrayView &a, const Scalar &otherwise) const { PlainObject r(a.m); for (int j = 0; j < cols; j++) for (int i = 0; i < rows; i++) if (!b[(size_t)j * rows + i]) r.ref(i, j) = otherwise; return r; }
  };
  ArrayView array() const { ArrayView v{PlainObject(*this)}; return v; }
  // diagonal matrix from a vector (eager)
  Matrix<Scalar, Dynamic, Dynamic> asDiagonal() const { Matrix<Scalar, Dynamic, Dynamic> d(size(), size()); d.setZero(); for (int i = 0; i < size(); i++) d.ref(i, i) = vget(i); return d; }
  Matrix<Scalar, (RowsAtCompileTime == 1 || ColsAtCompileTime == 1) ? Dynamic : RowsAtCompileTime, 1> diagonal() const {
    Matrix<Scalar, Dynamic, 1> d(std::min(rows(), cols())); for (int i = 0; i < d.rows(); i++) d.ref(i, 0) = coeff(i, i); return d; }
};

// ------------------------------------------------------------------------------------------------ Matrix
namespace shim {
template <class S, int R, int C, bool Fixed = (R != Dynamic && C != Dynamic)> struct Store;
template <class S, int R, int C> struct Store<S, R, C, true> {
  S d[R * C > 0 ? R * C : 1];
  Store() { for (int i = 0; i < R * C; i++) d[i] = S(0); }
  int r() const { return R; }
  int c() const { return C; }
  void resize(int rr, int cc) { (void)rr; (void)cc; assert(rr == R && cc == C); }
  S *p() { return d; }
  const S *p() const { return d; }
};
template <class S, int R, int C> struct Store<S, R, C, false> {
  std::vector<S> d; int nr, nc;
  Store() : nr(R == Dynamic ? 0 : R), nc(C == Dynamic ? 0 : C) {}
  int r() const { return nr; }
  int c() const { return nc; }
  void resize(int rr, int cc) { assert((R == Dynamic || rr == R) && (C == Dynamic || cc == C)); if (rr != nr || cc != nc) { nr = rr; nc = cc; d.assign((size_t)rr * cc, S(0)); } }
  S *p() { return d.data(); }
  const S *p() const { return d.data(); }
};
}  // namespace shim

template <class S, int R, int C, int Opt, int MR, int MC>
class Matrix : public MatrixBase<Matrix<S, R, C, Opt, MR, MC>> {
  shim::Store<S, R, C> st;
  typedef MatrixBase<Matrix> Base;
  enum { RowMaj = ((Opt & RowMajor) != 0) && R != 1 && C != 1 };

 public:
  typedef S Scalar;
  int rows_() const { return st.r(); }
  int cols_() const { return st.c(); }
  void resize_(int r, int c) { st.resize(r, c); }
  int idx(int i, int j) const { return RowMaj ? i * st.c() + j : j * st.r() + i; }
  S get(int i, int j) const { assert(i >= 0 && i < st.r() && j >= 0 && j < st.c()); return st.p()[idx(i, j)]; }
  S &ref(int i, int j) { assert(i >= 0 && i < st.r() && j >= 0 && j < st.c()); return st.p()[idx(i, j)]; }
  S *data() { return st.p(); }
  const S *data() const { return st.p(); }
  void resize(int r, int c) { st.resize(r, c); }
  void resize(int n) { if (C == 1) st.resize(n, 1); else st.resize(1, n); }
  void conservativeResize(int n) { if (C == 1) conservativeResize(n, 1); else conservativeResize(1, n); }
  void conservativeResize(int r, int c) { Matrix old(*this); st.resize(r, c); for (int j = 0; j < std::min(c, old.cols()); j++) for (int i = 0; i < std::min(r, old.rows()); i++) ref(i, j) = old.get(i, j); }

  Matrix() {}
  Matrix(const Matrix &o) = default;
  Matrix &operator=(const Matrix &o) = default;
  // (n) : dynamic vector size; a 1x1 fixed matrix takes it as the coefficient
  explicit Matrix(int n) { if (R == 1 && C == 1) st.p()[0] = S(n); else if (R == Dynamic && C == 1) st.resize(n, 1); else if (C == Dynamic && R == 1) st.resize(1, n); else if (R == Dynamic && C == Dynamic) st.resize(n, n); }
  template <class T0, class T1, class = typename std::enable_if<std::is_arithmetic<T0>::value && std::is_arithmetic<T1>::value>::type>
  Matrix(const T0 &a, const T1 &b) {
    if (R != Dynamic && C != Dynamic && R * C == 2) { st.p()[0] = S(a); st.p()[1] = S(b); }
    else st.resize((int)a, (int)b);
  }
  Matrix(const S &a, const S &b, const S &c) { st.resize(R == 1 ? 1 : 3, R == 1 ? 3 : 1); st.p()[0] = a; st.p()[1] = b; st.p()[2] = c; }
  Matrix(const S &a, const S &b, const S &c, const S &d) { st.resize(R == 1 ? 1 : 4, R == 1 ? 4 : 1); st.p()[0] = a; st.p()[1] = b; st.p()[2] = c; st.p()[3] = d; }
  template <class O> Matrix(const MatrixBase<O> &o) { st.resize(o.rows(), o.cols()); Base::assign(o); }
  template <class O> Matrix &operator=(const MatrixBase<O> &o) { Matrix tmp; tmp.st.resize(o.rows(), o.cols()); tmp.Base::assign(o); st = tmp.st; return *this; }

  static Matrix Zero() { Matrix m; return m; }
  static Matrix Zero(int r, int c) { Matrix m; m.st.resize(r, c); m.setZero(); return m; }
  static Matrix Zero(int n) { Matrix m(n); m.setZero(); return m; }
  static Matrix Identity() { Matrix m; m.setIdentity(); return m; }
  static Matrix Identity(int r, int c) { Matrix m; m.st.resize(r, c); m.setIdentity(); return m; }
  static Matrix Ones() { Matrix m; m.setConstant(S(1)); return m; }
  static Matrix Ones(int r, int c) { Matrix m; m.st.resize(r, c); m.setConstant(S(1)); return m; }
  static Matrix Constant(const S &v) { Matrix m; m.setConstant(v); return m; }
  static Matrix UnitX() { Matrix m; m.ref(0, 0) = S(1); return m; }
  static Matrix UnitY() { Matrix m; m.vref(1) = S(1); return m; }
  static Matrix UnitZ() { Matrix m; m.vref(2) = S(1); return m; }
};

// ------------------------------------------------------------------------------------------------ Block / Map
template <class X, int BR, int BC>
class Block : public MatrixBase<Block<X, BR, BC>> {
  X *x; int r0, c0, nr, nc;
  typedef MatrixBase<Block> Base;

 public:
  typedef typename traits<X>::Scalar Scalar;
  Block(X &xx, int i, int j, int r, int c) : x(&xx), r0(i), c0(j), nr(r), nc(c) { assert(i >= 0 && j >= 0 && i + r <= xx.rows() && j + c <= xx.cols()); }
  Block(const Block &) = default;
  int rows_() const { return nr; }
  int cols_() const { return nc; }
  void resize_(int r, int c) { (void)r; (void)c; assert(r == nr && c == nc); }
  Scalar get(int i, int j) const { return x->coeff(r0 + i, c0 + j); }
  Scalar &ref(int i, int j) { return const_cast<typename std::remove_const<X>::type *>(x)->coeffRef(r0 + i, c0 + j); }
  template <class O> Block &operator=(const MatrixBase<O> &o) { typename MatrixBase<O>::PlainObject tmp(o); Base::assign(tmp); return *this; }
  Block &operator=(const Block &o) { typename Base::PlainObject tmp(o); Base::assign(tmp); return *this; }
};

template <class M, int MapOpt, class Stride>
class Map : public MatrixBase<Map<M, MapOpt, Stride>> {
  typedef typename traits<M>::Scalar S;
  S *p; int nr, nc;
  typedef MatrixBase<Map> Base;
  enum { R = traits<M>::Rows, C = traits<M>::Cols, RowMaj = ((traits<M>::Options & RowMajor) != 0) && R != 1 && C != 1 };

 public:
  typedef S Scalar;
  Map(const S *ptr) : p(const_cast<S *>(ptr)), nr(R), nc(C) {}
  Map(const S *ptr, int n) : p(const_cast<S *>(ptr)), nr(C == 1 ? n : 1), nc(C == 1 ? 1 : n) {}
  Map(const S *ptr, int r, int c) : p(const_cast<S *>(ptr)), nr(r), nc(c) {}
  Map(const Map &) = default;
  int rows_() const { return nr; }
  int cols_() const { return nc; }
  void resize_(int r, int c) { (void)r; (void)c; assert(r == nr && c == nc); }
  S get(int i, int j) const { return p[RowMaj ? i * nc + j : j * nr + i]; }
  S &ref(int i, int j) { return p[RowMaj ? i * nc + j : j * nr + i]; }
  S *data() { return p; }
  const S *data() const { return p; }
  template <class O> Map &operator=(const MatrixBase<O> &o) { typename MatrixBase<O>::PlainObject tmp(o); Base::assign(tmp); return *this; }
  Map &operator=(const Map &o) { typename Base::PlainObject tmp(o); Base::assign(tmp); return *this; }
};

// ------------------------------------------------------------------------------------------------ operators
template <class A, class B>
Matrix<typename traits<A>::Scalar, shim::pick(traits<A>::Rows, traits<B>::Rows), shim::pick(traits<A>::Cols, traits<B>::Cols)>
operator+(const MatrixBase<A> &a, const MatrixBase<B> &b) {
  Matrix<typename traits<A>::Scalar, shim::pick(traits<A>::Rows, traits<B>::Rows), shim::pick(traits<A>::Cols, traits<B>::Cols)> r(a);
  assert(a.rows() == b.rows() && a.cols() == b.cols());
  for (int j = 0; j < a.cols(); j++) for (int i = 0; i < a.rows(); i++) r.ref(i, j) = a.coeff(i, j) + b.coeff(i, j);
  return r;
}
template <class A, class B>
Matrix<typename traits<A>::Scalar, shim::pick(traits<A>::Rows, traits<B>::Rows), shim::pick(traits<A>::Cols, traits<B>::Cols)>
operator-(const MatrixBase<A> &a, const MatrixBase<B> &b) {
  Matrix<typename traits<A>::Scalar, shim::pick(traits<A>::Rows, traits<B>::Rows), shim::pick(traits<A>::Cols, traits<B>::Cols)> r(a);
  assert(a.rows() == b.rows() && a.cols() == b.cols());
  for (int j = 0; j < a.cols(); j++) for (int i = 0; i < a.rows(); i++) r.ref(i, j) = a.coeff(i, j) - b.coeff(i, j);
  return r;
}
template <class A> typename MatrixBase<A>::PlainObject operator-(const MatrixBase<A> &a) {
  typename MatrixBase<A>::PlainObject r(a);
  for (int j = 0; j < a.cols(); j++) for (int i = 0; i < a.rows(); i++) r.ref(i, j) = -a.coeff(i, j);
  return r;
}
// matrix product: plain triple loop, k innermost and ascending (what Eigen's lazy coefficient-based product does for
// the small fixed sizes of the factor code: res(i,j) = sum_k lhs(i,k) * rhs(k,j))
template <class A, class B>
Matrix<typename traits<A>::Scalar, traits<A>::Rows, traits<B>::Cols> operator*(const MatrixBase<A> &a, const MatrixBase<B> &b) {
  typedef typename traits<A>::Scalar S;
  assert(a.cols() == b.rows());
  Matrix<S, traits<A>::Rows, traits<B>::Cols> r(a.rows(), b.cols());
  for (int i = 0; i < a.rows(); i++)
    for (int j = 0; j < b.cols(); j++) {
      S s = a.coeff(i, 0) * b.coeff(0, j);
      for (int k = 1; k < a.cols(); k++) s += a.coeff(i, k) * b.coeff(k, j);
      r.ref(i, j) = s;
    }
  return r;
}
template <class A> typename MatrixBase<A>::PlainObject operator*(const MatrixBase<A> &a, const typename traits<A>::Scalar &s) {
  typename MatrixBase<A>::PlainObject r(a);
  for (int j = 0; j < a.cols(); j++) for (int i = 0; i < a.rows(); i++) r.ref(i, j) = a.coeff(i, j) * s;
  return r;
}
template <class A> typename MatrixBase<A>::PlainObject operator*(const typename traits<A>::Scalar &s, const MatrixBase<A> &a) {
  typename MatrixBase<A>::PlainObject r(a);
  for (int j = 0; j < a.cols(); j++) for (int i = 0; i < a.rows(); i++) r.ref(i, j) = s * a.coeff(i, j);
  return r;
}
template <class A> typename MatrixBase<A>::PlainObject operator/(const MatrixBase<A> &a, const typename traits<A>::Scalar &s) {
  typename MatrixBase<A>::PlainObject r(a);
  for (int j = 0; j < a.cols(); j++) for (int i = 0; i < a.rows(); i++) r.ref(i, j) = a.coeff(i, j) / s;
  return r;
}
template <class A, class B> bool operator==(const MatrixBase<A> &a, const MatrixBase<B> &b) {
  if (a.rows() != b.rows() || a.cols() != b.cols()) return false;
  for (int j = 0; j < a.cols(); j++) for (int i = 0; i < a.rows(); i++) if (!(a.coeff(i, j) == b.coeff(i, j))) return false;
  return true;
}
template <class A, class B> bool operator!=(const MatrixBase<A> &a, const MatrixBase<B> &b) { return !(a == b); }
template <class A> std::ostream &operator<<(std::ostream &os, const MatrixBase<A> &a) {
  for (int i = 0; i < a.rows(); i++) { for (int j = 0; j < a.cols(); j++) os << (j ? " " : "") << a.coeff(i, j); if (i + 1 < a.rows()) os << "\n"; }
  return os;
}
template <class D> template <class O> void MatrixBase<D>::applyOnTheLeft(const MatrixBase<O> &m) { PlainObject t = m * (*this); assign(t); }
template <class D> template <class O> void MatrixBase<D>::applyOnTheRight(const MatrixBase<O> &m) { PlainObject t = (*this) * m; assign(t); }

namespace shim {
template <class D> struct CommaInit {
  D &m; int k;
  CommaInit(D &mm, const typename traits<D>::Scalar &v) : m(mm), k(0) { put(v); }
  void put(const typename traits<D>::Scalar &v) { int r = k / m.cols(), c = k % m.cols(); assert(r < m.rows()); m.coeffRef(r, c) = v; k++; }
  CommaInit &operator,(const typename traits<D>::Scalar &v) { put(v); return *this; }
  template <class O> CommaInit &operator,(const MatrixBase<O> &o) {   // only whole-row / column-vector fills are supported
    for (int j = 0; j < o.cols(); j++) for (int i = 0; i < o.rows(); i++) { if (m.cols() == 1) m.coeffRef(k + i, 0) = o.coeff(i, j); else m.coeffRef(k / m.cols() + i, k % m.cols() + j) = o.coeff(i, j); }
    k += m.cols() == 1 ? o.rows() : o.cols();
    return *this;
  }
};
}  // namespace shim
template <class D> shim::CommaInit<D> MatrixBase<D>::operator<<(const Scalar &v) { return shim::CommaInit<D>(derived(), v); }

// general inverse / determinant: Gauss-Jordan with partial pivoting (Eigen: closed forms up to 4x4, PartialPivLU above)
template <class D> typename MatrixBase<D>::PlainObject MatrixBase<D>::inverse() const {
  const int n = rows();
  assert(n == cols());
  std::vector<Scalar> a((size_t)n * 2 * n, Scalar(0));
  for (int i = 0; i < n; i++) { for (int j = 0; j < n; j++) a[(size_t)i * 2 * n + j] = coeff(i, j); a[(size_t)i * 2 * n + n + i] = Scalar(1); }
  for (int c = 0; c < n; c++) {
    int p = c;
    for (int i = c + 1; i < n; i++) if (std::fabs(a[(size_t)i * 2 * n + c]) > std::fabs(a[(size_t)p * 2 * n + c])) p = i;
    if (p != c) for (int j = 0; j < 2 * n; j++) std::swap(a[(size_t)p * 2 * n + j], a[(size_t)c * 2 * n + j]);
    const Scalar d = a[(size_t)c * 2 * n + c];
    for (int j = 0; j < 2 * n; j++) a[(size_t)c * 2 * n + j] /= d;
    for (int i = 0; i < n; i++) if (i != c) { const Scalar f = a[(size_t)i * 2 * n + c]; if (f != Scalar(0)) for (int j = 0; j < 2 * n; j++) a[(size_t)i * 2 * n + j] -= f * a[(size_t)c * 2 * n + j]; }
  }
  PlainObject r(n, n);
  for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) r.ref(i, j) = a[(size_t)i * 2 * n + n + j];
  return r;
}
template <class D> typename MatrixBase<D>::Scalar MatrixBase<D>::determinant() const {
  const int n = rows();
  std::vector<Scalar> a((size_t)n * n);
  for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) a[(size_t)i * n + j] = coeff(i, j);
  Scalar det = 1;
  for (int c = 0; c < n; c++) {
    int p = c;
    for (int i = c + 1; i < n; i++) if (std::fabs(a[(size_t)i * n + c]) > std::fabs(a[(size_t)p * n + c])) p = i;
    if (a[(size_t)p * n + c] == Scalar(0)) return Scalar(0);
    if (p != c) { for (int j = 0; j < n; j++) std::swap(a[(size_t)p * n + j], a[(size_t)c * n + j]); det = -det; }
    det *= a[(size_t)c * n + c];
    for (int i = c + 1; i < n; i++) { const Scalar f = a[(size_t)i * n + c] / a[(size_t)c * n + c]; for (int j = c; j < n; j++) a[(size_t)i * n + j] -= f * a[(size_t)c * n + j]; }
  }
  return det;
}

// ------------------------------------------------------------------------------------------------ decompositions
template <class M> class LLT {
  Matrix<typename traits<M>::Scalar, traits<M>::Rows, traits<M>::Cols> L; ComputationInfo inf;
 public:
  LLT() : inf(Success) {}
  template <class O> explicit LLT(const MatrixBase<O> &a) { compute(a); }
  template <class O> LLT &compute(const MatrixBase<O> &a) {
    typedef typename traits<M>::Scalar S;
    const int n = a.rows();
    L = a; inf = Success;
    for (int j = 0; j < n; j++) {
      S d = L(j, j);
      for (int k = 0; k < j; k++) d -= L(j, k) * L(j, k);
      if (!(d > S(0))) inf = NumericalIssue;
      d = std::sqrt(d); L(j, j) = d;
      for (int i = j + 1; i < n; i++) { S s = L(i, j); for (int k = 0; k < j; k++) s -= L(i, k) * L(j, k); L(i, j) = s / d; }
      for (int i = 0; i < j; i++) L(i, j) = S(0);
    }
    return *this;
  }
  const Matrix<typename traits<M>::Scalar, traits<M>::Rows, traits<M>::Cols> &matrixL() const { return L; }
  ComputationInfo info() const { return inf; }
};

template <class M> class SelfAdjointEigenSolver {   // cyclic Jacobi; eigenvalues ascending like Eigen
  typedef typename traits<M>::Scalar S;
  Matrix<S, traits<M>::Rows, traits<M>::Cols> V; Matrix<S, traits<M>::Rows, 1> ev; ComputationInfo inf;
 public:
  SelfAdjointEigenSolver() : inf(Success) {}
  template <class O> explicit SelfAdjointEigenSolver(const MatrixBase<O> &a) { compute(a); }
  template <class O> SelfAdjointEigenSolver &compute(const MatrixBase<O> &a0) {
    const int n = a0.rows();
    Matrix<S, Dynamic, Dynamic> A(a0); V = Matrix<S, traits<M>::Rows, traits<M>::Cols>::Identity(n, n);
    for (int sweep = 0; sweep < 100; sweep++) {
      S off = 0;
      for (int i = 0; i < n; i++) for (int j = i + 1; j < n; j++) off += A(i, j) * A(i, j);
      if (off < S(1e-300)) break;
      for (int p = 0; p < n; p++) for (int q = p + 1; q < n; q++) {
        const S apq = A(p, q);
        if (apq == S(0)) continue;
        const S tau = (A(q, q) - A(p, p)) / (S(2) * apq);
        const S t = (tau >= 0 ? S(1) : S(-1)) / (std::fabs(tau) + std::sqrt(S(1) + tau * tau));
        const S c = S(1) / std::sqrt(S(1) + t * t), s = t * c;
        for (int k = 0; k < n; k++) { const S x = A(k, p), y = A(k, q); A(k, p) = c * x - s * y; A(k, q) = s * x + c * y; }
        for (int k = 0; k < n; k++) { const S x = A(p, k), y = A(q, k); A(p, k) = c * x - s * y; A(q, k) = s * x + c * y; }
        for (int k = 0; k < n; k++) { const S x = V(k, p), y = V(k, q); V(k, p) = c * x - s * y; V(k, q) = s * x + c * y; }
      }
    }
    std::vector<int> ord(n); for (int i = 0; i < n; i++) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](int a, int b) { return A(a, a) < A(b, b); });
    Matrix<S, traits<M>::Rows, traits<M>::Cols> Vs(n, n); ev.resize_(n, 1);
    for (int j = 0; j < n; j++) { ev(j) = A(ord[j], ord[j]); for (int i = 0; i < n; i++) Vs(i, j) = V(i, ord[j]); }
    V = Vs; inf = Success;
    return *this;
  }
  const Matrix<S, traits<M>::Rows, 1> &eigenvalues() const { return ev; }
  const Matrix<S, traits<M>::Rows, traits<M>::Cols> &eigenvectors() const { return V; }
  ComputationInfo info() const { return inf; }
};

// JacobiSVD of a square matrix, full U and V, singular values descending like Eigen's: V = eigenvectors of A^T A (cyclic Jacobi
// above), sigma = sqrt of its eigenvalues, U = A V diag(1 / sigma), completed by Gram-Schmidt where sigma = 0.  (Eigen runs a
// two-sided Jacobi on A; both give the same factorisation up to the signs of paired columns and rounding.)
template <class M> class JacobiSVD {
  typedef typename traits<M>::Scalar S;
  M U, V; Matrix<S, traits<M>::Rows, 1> sv;
 public:
  template <class O> explicit JacobiSVD(const MatrixBase<O> &a0, int = 0) {
    const int n = a0.rows();
    assert(a0.cols() == n);
    Matrix<S, Dynamic, Dynamic> A(a0), AtA = Matrix<S, Dynamic, Dynamic>::Zero(n, n);
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) { S t = 0; for (int k = 0; k < n; k++) t += A(k, i) * A(k, j); AtA(i, j) = t; }
    SelfAdjointEigenSolver<Matrix<S, Dynamic, Dynamic>> es(AtA);
    U = M::Zero(n, n); V = M::Zero(n, n); sv.resize_(n, 1);
    for (int j = 0; j < n; j++) {
      const int c = n - 1 - j;   // eigenvalues ascending -> singular values descending
      const S l = es.eigenvalues()(c);
      sv(j) = l > S(0) ? std::sqrt(l) : S(0);
      for (int i = 0; i < n; i++) V(i, j) = es.eigenvectors()(i, c);
    }
    for (int j = 0; j < n; j++) {
      S nn = 0;
      for (int i = 0; i < n; i++) { S t = 0; for (int k = 0; k < n; k++) t += A(i, k) * V(k, j); U(i, j) = t; }
      if (sv(j) > S(0)) { for (int i = 0; i < n; i++) U(i, j) = U(i, j) / sv(j); continue; }
      for (int e = 0; e < n; e++) {   // Gram-Schmidt of a unit vector against the columns before j
        for (int i = 0; i < n; i++) U(i, j) = i == e ? S(1) : S(0);
        for (int p = 0; p < j; p++) { S d = 0; for (int i = 0; i < n; i++) d += U(i, p) * U(i, j); for (int i = 0; i < n; i++) U(i, j) -= d * U(i, p); }
        nn = 0; for (int i = 0; i < n; i++) nn += U(i, j) * U(i, j);
        if (nn > S(1e-6)) break;
      }
      for (int i = 0; i < n; i++) U(i, j) = U(i, j) / std::sqrt(nn);
    }
  }
  const M &matrixU() const { return U; }
  const M &matrixV() const { return V; }
  const Matrix<S, traits<M>::Rows, 1> &singularValues() const { return sv; }
};
template <class D> JacobiSVD<typename MatrixBase<D>::PlainObject> MatrixBase<D>::jacobiSvd(int opts) const {
  return JacobiSVD<PlainObject>(derived(), opts);
}

// "Sparse" types with Eigen's interface on DENSE storage (the marginalization code of the reference assembles its Jacobian
// from triplets and takes a sparse LLT; at oracle sizes a dense matrix computes the same numbers).
template <class S> struct Triplet {
  int r = 0, c = 0; S v = S(0);
  Triplet() {}
  Triplet(int r_, int c_, const S &v_) : r(r_), c(c_), v(v_) {}
  int row() const { return r; } int col() const { return c; } const S &value() const { return v; }
};
template <class S, int Opt = 0, class I = int> class SparseMatrix : public Matrix<S, Dynamic, Dynamic> {
  typedef Matrix<S, Dynamic, Dynamic> Dense;
 public:
  SparseMatrix() {}
  SparseMatrix(int r, int c) : Dense(Dense::Zero(r, c)) {}
  template <class O> SparseMatrix(const MatrixBase<O> &o) : Dense(o) {}
  template <class O> SparseMatrix &operator=(const MatrixBase<O> &o) { Dense::operator=(o); return *this; }
  template <class It> void setFromTriplets(It b, It e) { this->setZero(); for (It t = b; t != e; ++t) this->ref(t->row(), t->col()) += t->value(); }   // duplicates are summed
  Dense toDense() const { return Dense(*this); }
  int nonZeros() const { int n = 0; for (int j = 0; j < this->cols(); j++) for (int i = 0; i < this->rows(); i++) n += this->get(i, j) != S(0); return n; }
  int outerSize() const { return this->cols(); }
  class InnerIterator {   // the non-zero entries of column j, rows ascending
    const SparseMatrix &m; int j, i;
    void skip() { while (i < m.rows() && m.get(i, j) == S(0)) i++; }
   public:
    InnerIterator(const SparseMatrix &m_, int j_) : m(m_), j(j_), i(0) { skip(); }
    explicit operator bool() const { return i < m.rows(); }
    InnerIterator &operator++() { i++; skip(); return *this; }
    int row() const { return i; } int col() const { return j; } S value() const { return m.get(i, j); }
  };
};
template <class M, int UpLo = 1, class Ord = void> class SimplicialLLT {   // dense Cholesky behind the sparse-solver interface
  typedef typename M::Scalar S;
  Matrix<S, Dynamic, Dynamic> L; ComputationInfo inf = Success;
 public:
  SimplicialLLT() {}
  template <class O> explicit SimplicialLLT(const MatrixBase<O> &a) { compute(a); }
  template <class O> SimplicialLLT &compute(const MatrixBase<O> &a) {
    const int n = a.rows(); L = Matrix<S, Dynamic, Dynamic>::Zero(n, n); inf = Success;
    for (int j = 0; j < n; j++) {
      S d = a.coeff(j, j);
      for (int k = 0; k < j; k++) d -= L(j, k) * L(j, k);
      if (!(d > S(0))) { inf = NumericalIssue; return *this; }
      using std::sqrt; L(j, j) = sqrt(d);
      for (int i = j + 1; i < n; i++) { S t = a.coeff(i, j); for (int k = 0; k < j; k++) t -= L(i, k) * L(j, k); L(i, j) = t / L(j, j); }
    }
    return *this;
  }
  ComputationInfo info() const { return inf; }
  template <class O> Matrix<S, Dynamic, Dynamic> solve(const MatrixBase<O> &b) const {
    const int n = L.rows(); Matrix<S, Dynamic, Dynamic> x(b);
    for (int c = 0; c < x.cols(); c++) {
      for (int i = 0; i < n; i++) { S t = x(i, c); for (int k = 0; k < i; k++) t -= L(i, k) * x(k, c); x(i, c) = t / L(i, i); }
      for (int i = n - 1; i >= 0; i--) { S t = x(i, c); for (int k = i + 1; k < n; k++) t -= L(k, i) * x(k, c); x(i, c) = t / L(i, i); }
    }
    return x;
  }
};
template <class M, int UpLo = 1, class Ord = void> class SimplicialLDLT;
template <class T, int O = 0, class St = void> class Ref;
// Ref<const Matrix<..>>: binds to any expression of that shape; here a copy (the callers only read through it)
template <class S, int R, int C, int Opt, int MR, int MC, int O, class St>
class Ref<const Matrix<S, R, C, Opt, MR, MC>, O, St> : public Matrix<S, R, C, Opt, MR, MC> {
 public:
  template <class D> Ref(const MatrixBase<D> &m) : Matrix<S, R, C, Opt, MR, MC>(m) {}
};

// ------------------------------------------------------------------------------------------------ quaternions
template <class Derived> struct qtraits;
template <class S, int Opt> struct qtraits<Quaternion<S, Opt>> { typedef S Scalar; };
template <class S, int Opt, int MO, class St> struct qtraits<Map<Quaternion<S, Opt>, MO, St>> { typedef S Scalar; };
template <class S, int Opt, int MO, class St> struct qtraits<Map<const Quaternion<S, Opt>, MO, St>> { typedef S Scalar; };

template <class Derived>
class QuaternionBase {
 public:
  typedef typename qtraits<Derived>::Scalar Scalar;
  typedef Matrix<Scalar, 3, 1> Vector3;
  typedef Matrix<Scalar, 3, 3> Matrix3;
  const Scalar *c() const { return static_cast<const Derived *>(this)->cdata(); }
  Scalar *c() { return static_cast<Derived *>(this)->cdata(); }
  Scalar x() const { return c()[0]; }
  Scalar y() const { return c()[1]; }
  Scalar z() const { return c()[2]; }
  Scalar w() const { return c()[3]; }
  Scalar &x() { return c()[0]; }
  Scalar &y() { return c()[1]; }
  Scalar &z() { return c()[2]; }
  Scalar &w() { return c()[3]; }
  Vector3 vec() const { return Vector3(x(), y(), z()); }
  template <class T> Quaternion<T> cast() const { return Quaternion<T>(T(w()), T(x()), T(y()), T(z())); }
  Matrix<Scalar, 4, 1> coeffs() const { return Matrix<Scalar, 4, 1>(x(), y(), z(), w()); }
  Scalar squaredNorm() const { return x() * x() + y() * y() + z() * z() + w() * w(); }
  Scalar norm() const { using std::sqrt; return sqrt(squaredNorm()); }
  Quaternion<Scalar> conjugate() const { return Quaternion<Scalar>(w(), -x(), -y(), -z()); }
  Quaternion<Scalar> inverse() const {
    const Scalar n2 = squaredNorm();
    if (n2 > Scalar(0)) return Quaternion<Scalar>(w() / n2, -x() / n2, -y() / n2, -z() / n2);
    return Quaternion<Scalar>(Scalar(0), Scalar(0), Scalar(0), Scalar(0));
  }
  Quaternion<Scalar> normalized() const { const Scalar n = norm(); return Quaternion<Scalar>(w() / n, x() / n, y() / n, z() / n); }
  void normalize() { const Scalar n = norm(); x() /= n; y() /= n; z() /= n; w() /= n; }
  Derived &setIdentity() { x() = y() = z() = Scalar(0); w() = Scalar(1); return *static_cast<Derived *>(this); }
  template <class O> Scalar dot(const QuaternionBase<O> &o) const { return x() * o.x() + y() * o.y() + z() * o.z() + w() * o.w(); }
  // Hamilton product, term order of Eigen's generic quat_product
  template <class O> Quaternion<Scalar> operator*(const QuaternionBase<O> &b) const {
    const QuaternionBase &a = *this;
    return Quaternion<Scalar>(a.w() * b.w() - a.x() * b.x() - a.y() * b.y() - a.z() * b.z(),
                              a.w() * b.x() + a.x() * b.w() + a.y() * b.z() - a.z() * b.y(),
                              a.w() * b.y() + a.y() * b.w() + a.z() * b.x() - a.x() * b.z(),
                              a.w() * b.z() + a.z() * b.w() + a.x() * b.y() - a.y() * b.x());
  }
  // rotation of a vector: Eigen's _transformVector (uv = 2 v x p; p + w uv + v x uv)
  template <class O> Vector3 operator*(const MatrixBase<O> &p) const {
    const Vector3 v = vec(), pp(p(0), p(1), p(2));
    Vector3 uv = v.cross(pp);
    uv += uv;
    return pp + w() * uv + v.cross(uv);
  }
  Vector3 _transformVector(const Vector3 &p) const { return (*this) * p; }
  Matrix3 toRotationMatrix() const {
    Matrix3 res;
    const Scalar tx = Scalar(2) * x(), ty = Scalar(2) * y(), tz = Scalar(2) * z();
    const Scalar twx = tx * w(), twy = ty * w(), twz = tz * w();
    const Scalar txx = tx * x(), txy = ty * x(), txz = tz * x();
    const Scalar tyy = ty * y(), tyz = tz * y(), tzz = tz * z();
    res(0, 0) = Scalar(1) - (tyy + tzz); res(0, 1) = txy - twz; res(0, 2) = txz + twy;
    res(1, 0) = txy + twz; res(1, 1) = Scalar(1) - (txx + tzz); res(1, 2) = tyz - twx;
    res(2, 0) = txz - twy; res(2, 1) = tyz + twx; res(2, 2) = Scalar(1) - (txx + tyy);
    return res;
  }
  Matrix3 matrix() const { return toRotationMatrix(); }
  template <class O> Scalar angularDistance(const QuaternionBase<O> &o) const {
    Quaternion<Scalar> d = (*this) * o.conjugate();
    return Scalar(2) * std::atan2(d.vec().norm(), std::fabs(d.w()));
  }
};

template <class S, int Opt>
class Quaternion : public QuaternionBase<Quaternion<S, Opt>> {
  S q[4];
 public:
  typedef S Scalar;
  S *cdata() { return q; }
  const S *cdata() const { return q; }
  Quaternion() { q[0] = q[1] = q[2] = S(0); q[3] = S(1); }
  Quaternion(const S &w, const S &x, const S &y, const S &z) { q[0] = x; q[1] = y; q[2] = z; q[3] = w; }
  explicit Quaternion(const S *d) { for (int i = 0; i < 4; i++) q[i] = d[i]; }
  Quaternion(const Quaternion &) = default;
  Quaternion &operator=(const Quaternion &) = default;
  template <class O> Quaternion(const QuaternionBase<O> &o) { q[0] = o.x(); q[1] = o.y(); q[2] = o.z(); q[3] = o.w(); }
  template <class O> Quaternion &operator=(const QuaternionBase<O> &o) { q[0] = o.x(); q[1] = o.y(); q[2] = o.z(); q[3] = o.w(); return *this; }
  // from a rotation matrix (Shepperd's method as documented for Eigen)
  template <class O, class = typename std::enable_if<traits<O>::Rows == 3 && traits<O>::Cols == 3>::type>
  explicit Quaternion(const MatrixBase<O> &m) {
    S t = m(0, 0) + m(1, 1) + m(2, 2);
    if (t > S(0)) { t = std::sqrt(t + S(1)); q[3] = S(0.5) * t; t = S(0.5) / t; q[0] = (m(2, 1) - m(1, 2)) * t; q[1] = (m(0, 2) - m(2, 0)) * t; q[2] = (m(1, 0) - m(0, 1)) * t; }
    else {
      int i = 0; if (m(1, 1) > m(0, 0)) i = 1; if (m(2, 2) > m(i, i)) i = 2;
      const int j = (i + 1) % 3, k = (j + 1) % 3;
      t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + S(1));
      q[i] = S(0.5) * t; t = S(0.5) / t;
      q[3] = (m(k, j) - m(j, k)) * t; q[j] = (m(j, i) + m(i, j)) * t; q[k] = (m(k, i) + m(i, k)) * t;
    }
  }
  static Quaternion Identity() { return Quaternion(S(1), S(0), S(0), S(0)); }
  template <class A, class B> static Quaternion FromTwoVectors(const MatrixBase<A> &a, const MatrixBase<B> &b) {
    Matrix<S, 3, 1> v0 = a.normalized(), v1 = b.normalized();
    const S c = v1.dot(v0);
    if (c < S(-1) + S(1e-12)) { Matrix<S, 3, 1> ax = v0.cross(Matrix<S, 3, 1>(1, 0, 0)); if (ax.norm() < S(1e-6)) ax = v0.cross(Matrix<S, 3, 1>(0, 1, 0)); ax.normalize(); return Quaternion(S(0), ax(0), ax(1), ax(2)); }
    Matrix<S, 3, 1> axis = v0.cross(v1);
    const S s = std::sqrt((S(1) + c) * S(2)), invs = S(1) / s;
    return Quaternion(s * S(0.5), axis(0) * invs, axis(1) * invs, axis(2) * invs);
  }
};

template <class S, int Opt, int MO, class St>
class Map<Quaternion<S, Opt>, MO, St> : public QuaternionBase<Map<Quaternion<S, Opt>, MO, St>> {
  S *p;
 public:
  typedef S Scalar;
  explicit Map(S *ptr) : p(ptr) {}
  S *cdata() { return p; }
  const S *cdata() const { return p; }
  template <class O> Map &operator=(const QuaternionBase<O> &o) { const S a = o.x(), b = o.y(), c = o.z(), d = o.w(); p[0] = a; p[1] = b; p[2] = c; p[3] = d; return *this; }
  Map &operator=(const Map &o) { for (int i = 0; i < 4; i++) p[i] = o.p[i]; return *this; }
};
template <class S, int Opt, int MO, class St>
class Map<const Quaternion<S, Opt>, MO, St> : public QuaternionBase<Map<const Quaternion<S, Opt>, MO, St>> {
  const S *p;
 public:
  typedef S Scalar;
  explicit Map(const S *ptr) : p(ptr) {}
  S *cdata() { return const_cast<S *>(p); }
  const S *cdata() const { return p; }
};
template <class D> std::ostream &operator<<(std::ostream &os, const QuaternionBase<D> &q) { return os << q.x() << "i + " << q.y() << "j + " << q.z() << "k + " << q.w(); }

template <class S> class AngleAxis {
  S ang; Matrix<S, 3, 1> ax;
 public:
  template <class O> AngleAxis(const S &a, const MatrixBase<O> &axis) : ang(a), ax(axis) {}
  Matrix<S, 3, 3> toRotationMatrix() const {
    const S c = std::cos(ang), s = std::sin(ang), t = S(1) - c;
    Matrix<S, 3, 3> R;
    R(0, 0) = c + t * ax(0) * ax(0); R(0, 1) = t * ax(0) * ax(1) - s * ax(2); R(0, 2) = t * ax(0) * ax(2) + s * ax(1);
    R(1, 0) = t * ax(0) * ax(1) + s * ax(2); R(1, 1) = c + t * ax(1) * ax(1); R(1, 2) = t * ax(1) * ax(2) - s * ax(0);
    R(2, 0) = t * ax(0) * ax(2) - s * ax(1); R(2, 1) = t * ax(1) * ax(2) + s * ax(0); R(2, 2) = c + t * ax(2) * ax(2);
    return R;
  }
  operator Quaternion<S>() const { const S h = ang / S(2), s = std::sin(h); return Quaternion<S>(std::cos(h), s * ax(0), s * ax(1), s * ax(2)); }
};

// ------------------------------------------------------------------------------------------------ typedefs
#define SHIM_TYPEDEFS(S, SUF)                                                                          \
  typedef Matrix<S, 2, 2> Matrix2##SUF; typedef Matrix<S, 3, 3> Matrix3##SUF; typedef Matrix<S, 4, 4> Matrix4##SUF; \
  typedef Matrix<S, Dynamic, Dynamic> MatrixX##SUF; typedef Matrix<S, 2, 1> Vector2##SUF; typedef Matrix<S, 3, 1> Vector3##SUF; \
  typedef Matrix<S, 4, 1> Vector4##SUF; typedef Matrix<S, Dynamic, 1> VectorX##SUF; typedef Matrix<S, 1, 3> RowVector3##SUF; \
  typedef Matrix<S, 1, Dynamic> RowVectorX##SUF; typedef Matrix<S, 6, 6> Matrix6##SUF; typedef Matrix<S, 6, 1> Vector6##SUF;
SHIM_TYPEDEFS(double, d)
SHIM_TYPEDEFS(float, f)
SHIM_TYPEDEFS(int, i)
#undef SHIM_TYPEDEFS
typedef Quaternion<double> Quaterniond;
typedef Quaternion<float> Quaternionf;
typedef AngleAxis<double> AngleAxisd;
typedef Matrix<double, 3, 4> Matrix34d;
template <class T> using aligned_allocator = std::allocator<T>;
}  // namespace Eigen
#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
