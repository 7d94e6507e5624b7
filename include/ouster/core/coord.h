// coord.h -- core::Coord, Ray and BoundsF of zone monitoring (mirrors ouster_core/include/ouster/core/coord.h and
// ray.h; DESIGN f-8).  Eigen is absent (as in ouster/core/typedefs.h), so Coord is a three-float stand-in for
// Eigen::Vector3f with the operations zones use, evaluated in Eigen's order: a dot product is
// (x0 y0 + x1 y1) + x2 y2 and a cross product (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0).
#pragma once
#include <cmath>
#include <cstddef>
#include <utility>

namespace ouster {
namespace sdk {
namespace core {

struct Coord {
    float v[3] = {0.f, 0.f, 0.f};
    Coord() = default;
    Coord(float x, float y, float z) : v{x, y, z} {}
    explicit Coord(const float* p) : v{p[0], p[1], p[2]} {}
    float& operator[](size_t i) { return v[i]; }
    float operator[](size_t i) const { return v[i]; }
    float& operator()(size_t i) { return v[i]; }
    float operator()(size_t i) const { return v[i]; }
    float x() const { return v[0]; }
    float y() const { return v[1]; }
    float z() const { return v[2]; }
    Coord operator+(const Coord& o) const { return {v[0] + o.v[0], v[1] + o.v[1], v[2] + o.v[2]}; }
    Coord operator-(const Coord& o) const { return {v[0] - o.v[0], v[1] - o.v[1], v[2] - o.v[2]}; }
    Coord operator*(float s) const { return {v[0] * s, v[1] * s, v[2] * s}; }
    Coord operator/(float s) const { return {v[0] / s, v[1] / s, v[2] / s}; }
    Coord& operator+=(const Coord& o) {
        for (int k = 0; k < 3; ++k) v[k] += o.v[k];
        return *this;
    }
    float dot(const Coord& o) const { return (v[0] * o.v[0] + v[1] * o.v[1]) + v[2] * o.v[2]; }
    Coord cross(const Coord& o) const {
        return {v[1] * o.v[2] - v[2] * o.v[1], v[2] * o.v[0] - v[0] * o.v[2], v[0] * o.v[1] - v[1] * o.v[0]};
    }
    float squaredNorm() const { return dot(*this); }
    float norm() const { return std::sqrt(squaredNorm()); }
    Coord normalized() const {
        const float n = norm();
        return n > 0.f ? *this / n : *this;
    }
    bool operator==(const Coord& o) const { return v[0] == o.v[0] && v[1] == o.v[1] && v[2] == o.v[2]; }
    bool operator!=(const Coord& o) const { return !(*this == o); }
};

/// A beam: origin and direction (ray.h).
struct Ray {
    Coord offset;
    Coord direction;
};

/// (near, far) distances along a ray.
using BoundsF = std::pair<float, float>;

}  // namespace core
}  // namespace sdk
}  // namespace ouster
