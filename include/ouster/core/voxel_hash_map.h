// voxel_hash_map.h -- voxel-grid downsampling (mirrors the free functions of
// ouster_core/include/ouster/core/voxel_hash_map.h:685-711 and ouster_core/src/voxel_hash_map.cpp:262-393;
// SURVEY 8f #2).  Same names, defaults and exception texts; the work runs on the GPU (ob_voxel_downsample,
// ouster-sdk_b200/csrc/ob_voxel.cu).
//
// Not part of this replacement: the VoxelHashMap class template itself (incremental add_points / update,
// get_closest_neighbor, remove_voxels_far_from_location, the bucket and strategy types) and
// IndexedVoxelHashMap3d -- only the one-shot downsampling functions are.
//
// Differences a caller can see:
//  * the reference's std::vector<Eigen::Vector3d> / ArrayX3dR arguments are n x 3 (n x d) row-major
//    ArrayRef<const double> views, results are DenseArray<double> (as in pose_util.h);
//  * voxel_downsample_3d / _xd emit voxels in the order of their first input row; the reference emits them
//    in tsl::robin_map iteration order (DESIGN 9).  voxel_downsample's order and indices are the reference's.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/typedefs.h"

namespace ouster {
namespace sdk {
namespace core {

/// voxel_hash_map.h:697-701
enum class VoxelDownsampleStrategy {
    FIRST_N_POINT,  ///< first n points of a voxel (n = max_points_per_voxel), no two closer than voxel_size/sqrt(n)
    AVERAGE_POINT,  ///< per-voxel average of every column
    RANDOM,         ///< random replacement once a voxel holds max_points_per_voxel points
};

namespace impl {
/// One call of the C ABI on the calling thread's stream; returns the number of output rows.
inline size_t run_voxel_downsample(int mode, const double* points, size_t n, size_t cols, const double* normals,
                                   double voxel_size, size_t max_points_per_voxel, size_t min_pts_threshold,
                                   double* out, double* normals_out, uint32_t* indices_out) {
    ob_voxel_io io{};
    io.mode = mode;
    io.dtype = OB_F64;
    io.points = points;
    io.cols = cols;
    io.normals = normals;
    io.n = n;
    io.voxel_size = voxel_size;
    io.max_points_per_voxel = max_points_per_voxel;
    io.min_pts_threshold = min_pts_threshold;
    io.points_out = out;
    io.normals_out = normals_out;
    io.indices_out = indices_out;
    size_t n_out = 0;
    io.n_out = &n_out;
    b200::check(ob_voxel_downsample(&io, b200::thread_stream()));
    return n_out;
}

inline DenseArray<double> first_rows(const DenseArray<double>& a, size_t rows) {
    DenseArray<double> out(rows, a.cols());
    for (size_t i = 0; i < rows * a.cols(); ++i) out.data()[i] = a.data()[i];
    return out;
}

inline DenseArray<double> voxel_downsample_nd(const ArrayRef<const double>& frame, double voxel_size,
                                              size_t max_points_per_voxel, size_t min_pts_threshold,
                                              VoxelDownsampleStrategy strategy, const char* name) {
    int mode = -1;
    switch (strategy) {
        case VoxelDownsampleStrategy::FIRST_N_POINT: mode = OB_VOXEL_FIRST_N_POINT; break;
        case VoxelDownsampleStrategy::AVERAGE_POINT: mode = OB_VOXEL_AVERAGE_POINT; break;
        case VoxelDownsampleStrategy::RANDOM: mode = OB_VOXEL_RANDOM; break;
    }
    if (mode < 0) throw std::invalid_argument(std::string(name) + ": unknown strategy");
    DenseArray<double> out(frame.rows(), frame.cols());
    const size_t m = run_voxel_downsample(mode, frame.data(), frame.rows(), frame.cols(), nullptr, voxel_size,
                                          max_points_per_voxel, min_pts_threshold, out.data(), nullptr, nullptr);
    return first_rows(out, m);
}
}  // namespace impl

/// voxel_downsample(frame, voxel_size) (voxel_hash_map.cpp:262-310): Fisher-Yates shuffle (xorshift32, seed 42),
/// then the first point of every voxel in shuffled order.  frame: n x 3.  Returns (points m x 3, source indices);
/// output order and indices are exactly the reference's.  voxel_size is not validated.
inline std::pair<DenseArray<double>, std::vector<uint32_t>> voxel_downsample(const ArrayRef<const double>& frame,
                                                                             const double voxel_size) {
    const size_t n = frame.rows();
    if (n == 0) return {DenseArray<double>(0, 3), {}};
    if (frame.cols() != 3) throw std::invalid_argument("voxel_downsample: points must be Nx3");
    DenseArray<double> out(n, 3);
    std::vector<uint32_t> idx(n);
    const size_t m = impl::run_voxel_downsample(OB_VOXEL_SHUFFLE_FIRST, frame.data(), n, 3, nullptr, voxel_size, 1, 1,
                                                out.data(), nullptr, idx.data());
    idx.resize(m);
    return {impl::first_rows(out, m), std::move(idx)};
}

/// voxel_downsample_3d(frame, voxel_size, max_points_per_voxel = 1, min_pts_threshold = 1, strategy = RANDOM)
/// (voxel_hash_map.cpp:312-348): frame n x 3.  min_pts_threshold applies to AVERAGE_POINT only.
/// @throws std::invalid_argument "max_points_per_voxel must be greater than 0", "voxel_size must be greater
/// than 0", "voxel_downsample_3d: unknown strategy" (an empty frame returns before any check).
inline DenseArray<double> voxel_downsample_3d(const ArrayRef<const double>& frame, const double voxel_size,
                                              const size_t max_points_per_voxel = 1,
                                              const size_t min_pts_threshold = 1,
                                              const VoxelDownsampleStrategy strategy = VoxelDownsampleStrategy::RANDOM) {
    if (frame.rows() == 0) return DenseArray<double>(0, 3);
    if (frame.cols() != 3) throw std::invalid_argument("voxel_downsample_3d: frame must be Nx3");
    return impl::voxel_downsample_nd(frame, voxel_size, max_points_per_voxel, min_pts_threshold, strategy,
                                     "voxel_downsample_3d");
}

/// voxel_downsample_xd(frame, ...) (voxel_hash_map.cpp:350-393): frame n x d, d >= 3; the voxel comes from
/// columns 0-2, the other columns are carried along (averaged for AVERAGE_POINT).
/// @throws additionally std::invalid_argument "voxel_downsample_xd: frame must have at least 3 columns".
inline DenseArray<double> voxel_downsample_xd(const ArrayRef<const double>& frame, const double voxel_size,
                                              const size_t max_points_per_voxel = 1,
                                              const size_t min_pts_threshold = 1,
                                              const VoxelDownsampleStrategy strategy = VoxelDownsampleStrategy::RANDOM) {
    if (frame.rows() == 0) return DenseArray<double>(0, frame.cols());
    if (frame.cols() < 3) throw std::invalid_argument("voxel_downsample_xd: frame must have at least 3 columns");
    return impl::voxel_downsample_nd(frame, voxel_size, max_points_per_voxel, min_pts_threshold, strategy,
                                     "voxel_downsample_xd");
}

}  // namespace core
}  // namespace sdk
}  // namespace ouster
