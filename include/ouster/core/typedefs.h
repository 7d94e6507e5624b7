// typedefs.h -- dense row-major containers used by the hot-path API.
//
// The reference (ouster_core/include/ouster/core/typedefs.h:57-176) aliases Eigen types:
//   img_t<T>         = Eigen::Array<T, Dynamic, Dynamic, RowMajor>
//   ArrayX3R<T>      = Eigen::Array<T, Dynamic, 3, RowMajor>
//   PointCloudXYZ<T> = Eigen::Array<T, Dynamic, 3, RowMajor>
// and passes them as Eigen::Ref.  Eigen is used on this path only as a typed pointer carrier
// (SURVEY 1), so the replacement ships a minimal owning array (DenseArray) and a non-owning
// view (ArrayRef) with the same memory layout (dense, row-major) and the same accessor names
// (.data() .rows() .cols() .size() operator()(r,c)).  With Eigen present an Eigen::Ref adapts
// to ArrayRef without a copy.
#pragma once
#include <algorithm>
#include <array>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <type_traits>
#include <vector>

namespace ouster {
namespace sdk {
namespace core {

template <typename T>
class ArrayRef;

/// Owning dense row-major rows x cols array.
template <typename T>
class DenseArray {
   public:
    using Scalar = T;
    DenseArray() = default;
    DenseArray(size_t rows, size_t cols) : rows_(rows), cols_(cols), buf_(rows * cols) {}
    static DenseArray Zero(size_t rows, size_t cols) { return DenseArray(rows, cols); }
    T* data() { return buf_.data(); }
    const T* data() const { return buf_.data(); }
    size_t rows() const { return rows_; }
    size_t cols() const { return cols_; }
    size_t size() const { return rows_ * cols_; }
    T& operator()(size_t r, size_t c) { return buf_[r * cols_ + c]; }
    const T& operator()(size_t r, size_t c) const { return buf_[r * cols_ + c]; }
    T& operator()(size_t i) { return buf_[i]; }
    const T& operator()(size_t i) const { return buf_[i]; }
    void setZero() { std::fill(buf_.begin(), buf_.end(), T{}); }
    void setConstant(const T& v) { std::fill(buf_.begin(), buf_.end(), v); }
    void resize(size_t rows, size_t cols) {
        rows_ = rows;
        cols_ = cols;
        buf_.assign(rows * cols, T{});
    }
    bool operator==(const DenseArray& o) const {
        return rows_ == o.rows_ && cols_ == o.cols_ && buf_ == o.buf_;
    }
    bool operator!=(const DenseArray& o) const { return !(*this == o); }
    template <typename U>
    DenseArray<U> cast() const {
        DenseArray<U> out(rows_, cols_);
        for (size_t i = 0; i < buf_.size(); ++i) out(i) = static_cast<U>(buf_[i]);
        return out;
    }

   private:
    size_t rows_{0}, cols_{0};
    std::vector<T> buf_;
};

/// Non-owning view of a dense row-major array (the role Eigen::Ref plays in the reference).
template <typename T>
class ArrayRef {
   public:
    using Scalar = typename std::remove_const<T>::type;
    ArrayRef() = default;
    ArrayRef(T* data, size_t rows, size_t cols) : data_(data), rows_(rows), cols_(cols) {}
    ArrayRef(DenseArray<Scalar>& a) : data_(a.data()), rows_(a.rows()), cols_(a.cols()) {}
    template <typename U = T, typename = typename std::enable_if<std::is_const<U>::value>::type>
    ArrayRef(const DenseArray<Scalar>& a) : data_(a.data()), rows_(a.rows()), cols_(a.cols()) {}
    template <typename U = T, typename = typename std::enable_if<std::is_const<U>::value>::type>
    ArrayRef(const ArrayRef<Scalar>& a) : data_(a.data()), rows_(a.rows()), cols_(a.cols()) {}
    T* data() const { return data_; }
    size_t rows() const { return rows_; }
    size_t cols() const { return cols_; }
    size_t size() const { return rows_ * cols_; }
    T& operator()(size_t r, size_t c) const { return data_[r * cols_ + c]; }
    T& operator()(size_t i) const { return data_[i]; }

   private:
    T* data_{nullptr};
    size_t rows_{0}, cols_{0};
};

template <typename T>
using img_t = DenseArray<T>;
template <typename T>
using ArrayX3R = DenseArray<T>;  ///< n x 3 row-major
template <typename T>
using PointCloudXYZ = DenseArray<T>;  ///< n x 3 row-major
using PointCloudXYZd = PointCloudXYZ<double>;
using PointCloudXYZf = PointCloudXYZ<float>;

/// 4x4 row-major double matrix (stand-in for Eigen's mat4d).
struct mat4d {
    std::array<double, 16> m{};
    mat4d() = default;
    static mat4d Identity() {
        mat4d r;
        for (int i = 0; i < 4; ++i) r.m[i * 4 + i] = 1.0;
        return r;
    }
    double& operator()(int r, int c) { return m[r * 4 + c]; }
    const double& operator()(int r, int c) const { return m[r * 4 + c]; }
    const double* data() const { return m.data(); }
    mat4d operator*(const mat4d& o) const {
        mat4d r;
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) {
                double s = 0;
                for (int k = 0; k < 4; ++k) s += m[i * 4 + k] * o.m[k * 4 + j];
                r.m[i * 4 + j] = s;
            }
        return r;
    }
    bool operator==(const mat4d& o) const { return m == o.m; }
};

/// Row-major 4x4 pose (stand-in for Eigen::Matrix<double, 4, 4, RowMajor>, typedefs.h Matrix4dR).
using Matrix4dR = mat4d;

/// 3-vector of doubles (stand-in for Eigen::Vector3d): three contiguous doubles, so a std::vector<Vector3d> is an
/// n x 3 row-major array.
struct Vector3d {
    double v[3] = {0.0, 0.0, 0.0};
    Vector3d() = default;
    Vector3d(double x, double y, double z) : v{x, y, z} {}
    double& operator[](int i) { return v[i]; }
    const double& operator[](int i) const { return v[i]; }
    double& operator()(int i) { return v[i]; }
    const double& operator()(int i) const { return v[i]; }
    double x() const { return v[0]; }
    double y() const { return v[1]; }
    double z() const { return v[2]; }
    double* data() { return v; }
    const double* data() const { return v; }
    bool operator==(const Vector3d& o) const { return v[0] == o.v[0] && v[1] == o.v[1] && v[2] == o.v[2]; }
};
static_assert(sizeof(Vector3d) == 3 * sizeof(double), "Vector3d must be three packed doubles");

}  // namespace core
}  // namespace sdk
}  // namespace ouster
