// voxel_downsample.h -- voxel-grid downsampling of points with normals (mirrors
// ouster_algorithm/include/ouster/algorithm/voxel_downsample.h and ouster_algorithm/src/voxel_downsample.cpp:21-57;
// SURVEY 8f #2).  Same name, argument meaning and exception texts; the work runs on the GPU
// (ob_voxel_downsample, mode OB_VOXEL_POINT_NORMAL).  Voxels come out in the order of their first accepted row
// (the reference: tsl::robin_map iteration order, DESIGN 9).
#pragma once
#include <stdexcept>
#include <utility>

#include "ouster/core/voxel_hash_map.h"

namespace ouster {
namespace sdk {
namespace algorithm {

/// voxel_downsample_with_normals(points, normals, voxel_size): rows with a non-finite point or normal, or a
/// normal of norm <= 1e-12, are skipped; per voxel the positions are averaged and the unit normals summed and
/// renormalised (a voxel whose sum has norm <= 1e-12 is dropped).  Returns (points m x 3, normals m x 3).
/// @throws std::invalid_argument "voxel_downsample_with_normals expects Nx3 inputs",
/// "voxel_downsample_with_normals points/normals size mismatch", "voxel_downsample_with_normals voxel_size must be > 0".
inline std::pair<core::DenseArray<double>, core::DenseArray<double>> voxel_downsample_with_normals(
    const core::ArrayRef<const double>& points, const core::ArrayRef<const double>& normals, double voxel_size) {
    if (points.cols() != 3 || normals.cols() != 3)
        throw std::invalid_argument("voxel_downsample_with_normals expects Nx3 inputs");
    if (points.rows() != normals.rows())
        throw std::invalid_argument("voxel_downsample_with_normals points/normals size mismatch");
    if (!(voxel_size > 0.0)) throw std::invalid_argument("voxel_downsample_with_normals voxel_size must be > 0");
    const size_t n = points.rows();
    core::DenseArray<double> p(n, 3), q(n, 3);
    const size_t m = core::impl::run_voxel_downsample(OB_VOXEL_POINT_NORMAL, points.data(), n, 3, normals.data(),
                                                      voxel_size, 1, 1, p.data(), q.data(), nullptr);
    return {core::impl::first_rows(p, m), core::impl::first_rows(q, m)};
}

}  // namespace algorithm
}  // namespace sdk
}  // namespace ouster
