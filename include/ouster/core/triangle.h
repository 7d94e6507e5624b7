// triangle.h -- core::Triangle (mirrors ouster_core/include/ouster/core/triangle.h and src/triangle.cpp:13-50;
// DESIGN f-8).  intersect() is the host form of the test the GPU renderer runs for every pixel (ob_zone.cu); it is
// here for callers that test single rays.  Compile without FMA contraction (-ffp-contract=off) to get the
// renderer's float results bit for bit.
#pragma once
#include <cmath>
#include <limits>

#include "ouster/core/coord.h"

namespace ouster {
namespace sdk {
namespace core {

struct Triangle {
    Coord coords[3];
    Coord edges[3];  ///< b - a, c - b, a - c
    Coord normal;    ///< unit normal of edges[0] x edges[1]

    Triangle(const Coord& a, const Coord& b, const Coord& c)
        : coords{a, b, c}, edges{b - a, c - b, a - c}, normal{edges[0].cross(edges[1]).normalized()} {}

    /// Distance along the ray to the triangle (Moller-Trumbore with edges from coords[0]), or
    /// std::numeric_limits<float>::lowest() for a ray parallel to it (|det| < epsilon) or one that passes outside
    /// it.  Barycentric bounds allow epsilon of slack.  A NaN passes every test and comes back as a NaN distance.
    float intersect(const Ray& beam) const {
        const float eps = std::numeric_limits<float>::epsilon();
        const float miss = std::numeric_limits<float>::lowest();
        const Coord e1 = coords[1] - coords[0];
        const Coord e2 = coords[2] - coords[0];
        const Coord p = beam.direction.cross(e2);
        const float det = e1.dot(p);
        if (det > -eps && det < eps) return miss;
        const float inv = 1.0f / det;
        const Coord s = beam.offset - coords[0];
        const float u = inv * s.dot(p);
        if ((u < 0 && std::fabs(u) > eps) || (u > 1 && std::fabs(u - 1) > eps)) return miss;
        const Coord q = s.cross(e1);
        const float v = inv * beam.direction.dot(q);
        if ((v < 0 && std::fabs(v) > eps) || (u + v > 1 && std::fabs(u + v - 1) > eps)) return miss;
        return inv * e2.dot(q);
    }

    bool operator==(const Triangle& o) const {
        return coords[0] == o.coords[0] && coords[1] == o.coords[1] && coords[2] == o.coords[2];
    }
};

}  // namespace core
}  // namespace sdk
}  // namespace ouster
