// normals.h -- surface normals on destaggered point clouds
// (mirrors ouster_algorithm/include/ouster/algorithm/normals.h:19-113; SURVEY 8f #2).  Same names,
// argument meaning, defaults and exception texts; the stencil runs on the GPU (ob_normals,
// ouster-sdk_b200/csrc/ob_normals.cu).
#pragma once
#include <cmath>
#include <stdexcept>
#include <utility>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/typedefs.h"

namespace ouster {
namespace sdk {
namespace algorithm {

/// Default target neighbour distance in meters (25 mm).
constexpr double DEFAULT_TARGET_DISTANCE_METER = 0.025;
/// Default minimum incidence angle (1 deg, ~0.01745 rad) used for AOI gating.
constexpr double DEFAULT_MIN_ANGLE_INCIDENCE_RAD = 1 * 3.14159265358979323846 / 180.0;

namespace impl {
inline void run_normals(const core::ArrayRef<const double>& xyz, const core::ArrayRef<const uint32_t>& range,
                        const double* xyz2, const uint32_t* range2, const core::ArrayRef<const double>& origins,
                        double* n1, double* n2, size_t pixel_search_range, double min_angle_of_incidence_rad,
                        double target_distance_m) {
    ob_normals_io io{};
    io.n_frames = 1;
    io.h = range.rows();
    io.w = range.cols();
    io.xyz = xyz.data();
    io.range = range.data();
    io.xyz2 = xyz2;
    io.range2 = range2;
    io.normals = n1;
    io.normals2 = n2;
    io.sensor_origins_xyz = origins.data();
    io.n_origins = origins.rows();
    io.pixel_search_range = pixel_search_range;
    io.min_angle_of_incidence_rad = min_angle_of_incidence_rad;
    io.target_distance_m = target_distance_m;
    core::b200::check(ob_normals(OB_F64, &io, core::b200::thread_stream()));
    core::b200::synchronize();
}
}  // namespace impl

/// normals(xyz, range, sensor_origins_xyz, ...): single return (normals.h:58-64, normals.cpp:411-430).
/// xyz: destaggered (H*W, 3); range: destaggered (H, W); sensor_origins_xyz: (W, 3).
/// @throws std::runtime_error "normals: xyz dimensions mismatch", "normals: sensor_origins size must
/// match image width", "normals: target_distance_m must be positive", "normals:
/// min_angle_of_incidence_rad must be positive".
inline core::DenseArray<double> normals(const core::ArrayRef<const double>& xyz,
                                        const core::ArrayRef<const uint32_t>& range,
                                        const core::ArrayRef<const double>& sensor_origins_xyz,
                                        size_t pixel_search_range = 1,
                                        double min_angle_of_incidence_rad = DEFAULT_MIN_ANGLE_INCIDENCE_RAD,
                                        double target_distance_m = DEFAULT_TARGET_DISTANCE_METER) {
    const size_t h = range.rows(), w = range.cols();
    if (xyz.rows() != h * w || xyz.cols() != 3) throw std::runtime_error("normals: xyz dimensions mismatch");
    if (sensor_origins_xyz.rows() != w)
        throw std::runtime_error("normals: sensor_origins size must match image width");
    core::DenseArray<double> out(h * w, 3);
    impl::run_normals(xyz, range, nullptr, nullptr, sensor_origins_xyz, out.data(), nullptr, pixel_search_range,
                      min_angle_of_incidence_rad, target_distance_m);
    return out;
}

/// Dual-return overload (normals.h:100-108, normals.cpp:432-483): the returns see each other's points as
/// neighbours; the second uses the first's vertical pixel subtent when that is > 0, else derives its own.
/// @throws additionally std::runtime_error "normals: range2 dimensions mismatch".
inline std::pair<core::DenseArray<double>, core::DenseArray<double>> normals(
    const core::ArrayRef<const double>& xyz, const core::ArrayRef<const uint32_t>& range,
    const core::ArrayRef<const double>& xyz2, const core::ArrayRef<const uint32_t>& range2,
    const core::ArrayRef<const double>& sensor_origins_xyz, size_t pixel_search_range = 1,
    double min_angle_of_incidence_rad = DEFAULT_MIN_ANGLE_INCIDENCE_RAD,
    double target_distance_m = DEFAULT_TARGET_DISTANCE_METER) {
    const size_t h = range.rows(), w = range.cols();
    if (xyz.rows() != h * w || xyz.cols() != 3 || xyz2.rows() != h * w || xyz2.cols() != 3)
        throw std::runtime_error("normals: xyz dimensions mismatch");
    if (range2.rows() != h || range2.cols() != w) throw std::runtime_error("normals: range2 dimensions mismatch");
    if (sensor_origins_xyz.rows() != w)
        throw std::runtime_error("normals: sensor_origins size must match image width");
    core::DenseArray<double> first(h * w, 3), second(h * w, 3);
    impl::run_normals(xyz, range, xyz2.data(), range2.data(), sensor_origins_xyz, first.data(), second.data(),
                      pixel_search_range, min_angle_of_incidence_rad, target_distance_m);
    return {std::move(first), std::move(second)};
}

}  // namespace algorithm
}  // namespace sdk
}  // namespace ouster
