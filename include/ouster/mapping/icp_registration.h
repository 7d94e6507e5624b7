// icp_registration.h -- ICPRegistration and build_linear_system (mirrors
// ouster_mapping/include/ouster/mapping/icp_registration.h and ouster_mapping/src/icp_registration.cpp; DESIGN f-6).
// Same names, defaults and public fields; the iterations run on the GPU (ob_icp_align, ob_icp_linear_system,
// ouster-sdk_b200/csrc/ob_voxel_map.cu) against a device-resident core::VoxelHashMap3d or core::VoxelHashMapXd.
//
// Eigen is absent (as in ouster/core/typedefs.h): Matrix6d / Vector6d are plain row-major arrays with the accessor
// names the reference's callers use, Correspondences is a vector of (source, target) core::Vector3d pairs.
//
// Differences a caller can see:
//  * build_linear_system's JtJ has the reference's lower triangle filled and the strict upper triangle zero, as the
//    reference leaves it; the sums follow parallel_deterministic_reduce's tree, so they are the reference's bit for
//    bit (DESIGN 4);
//  * align_points_to_map's pose agrees with a CPU restatement to about 1e-12: device sin/cos are not host libm
//    (DESIGN 9);
//  * max_num_threads_ only reads back (the hardware concurrency when 0 is given); it has no effect on the GPU.
#pragma once
#include <array>
#include <thread>
#include <utility>
#include <vector>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/typedefs.h"
#include "ouster/core/voxel_hash_map.h"

namespace ouster {
namespace sdk {
namespace mapping {

/// 6x6 row-major double matrix (stand-in for Eigen::Matrix<double, 6, 6>)
struct Matrix6d {
    std::array<double, 36> m{};
    static Matrix6d Zero() { return Matrix6d(); }
    double& operator()(int r, int c) { return m[r * 6 + c]; }
    const double& operator()(int r, int c) const { return m[r * 6 + c]; }
    double* data() { return m.data(); }
    const double* data() const { return m.data(); }
};
/// 6-vector of doubles (stand-in for Eigen::Matrix<double, 6, 1>)
struct Vector6d {
    std::array<double, 6> v{};
    static Vector6d Zero() { return Vector6d(); }
    double& operator()(int i) { return v[i]; }
    const double& operator()(int i) const { return v[i]; }
    double& operator[](int i) { return v[i]; }
    const double& operator[](int i) const { return v[i]; }
    double* data() { return v.data(); }
    const double* data() const { return v.data(); }
};
using Correspondences = std::vector<std::pair<core::Vector3d, core::Vector3d>>;
using LinearSystem = std::pair<Matrix6d, Vector6d>;

/// build_linear_system(correspondences, kernel_scale) (icp_registration.cpp): Geman-McClure weighted JtJ (lower
/// triangle) and Jtr over the pairs (source, target), summed in parallel_deterministic_reduce's tree (grain 128).
inline LinearSystem build_linear_system(const Correspondences& correspondences, const double kernel_scale) {
    std::vector<double> src(correspondences.size() * 3), tgt(correspondences.size() * 3);
    for (size_t i = 0; i < correspondences.size(); ++i)
        for (int d = 0; d < 3; ++d) {
            src[3 * i + d] = correspondences[i].first[d];
            tgt[3 * i + d] = correspondences[i].second[d];
        }
    LinearSystem out;
    ob_icp_system_io io{};
    io.source = src.data();
    io.target = tgt.data();
    io.n = correspondences.size();
    io.kernel_scale = kernel_scale;
    io.jtj = out.first.data();
    io.jtr = out.second.data();
    core::b200::check(ob_icp_linear_system(&io, core::b200::thread_stream()));
    return out;
}

/// ICPRegistration (icp_registration.h): point-to-point ICP with a Geman-McClure kernel against a VoxelHashMap3d or a
/// VoxelHashMapXd (which it reads x, y, z of only).
struct ICPRegistration {
    explicit ICPRegistration(int max_num_iteration = 50, double convergence_criterion = 0.0001,
                             int max_num_threads = 0)
        : max_num_iterations_(max_num_iteration),
          convergence_criterion_(convergence_criterion),
          max_num_threads_(max_num_threads > 0 ? max_num_threads
                                               : static_cast<int>(std::thread::hardware_concurrency() > 0
                                                                      ? std::thread::hardware_concurrency()
                                                                      : 1)) {}

    /// align_points_to_map(frame, voxel_map, max_distance, kernel_scale): the correction that moves `frame` onto
    /// the map; the identity for an empty map.
    core::Matrix4dR align_points_to_map(const std::vector<core::Vector3d>& frame, const core::VoxelHashMap3d& voxel_map,
                                        const double max_distance, const double kernel_scale) const {
        return align(frame, voxel_map, max_distance, kernel_scale);
    }
    /// align_points_to_map(frame, VoxelHashMapXd, max_distance, kernel_scale) (icp_registration.cpp:205-210): the
    /// same iterations on the map's x, y, z; the pose is the one a VoxelHashMap3d of the same x, y, z gives
    core::Matrix4dR align_points_to_map(const std::vector<core::Vector3d>& frame, const core::VoxelHashMapXd& voxel_map,
                                        const double max_distance, const double kernel_scale) const {
        return align(frame, voxel_map, max_distance, kernel_scale);
    }

    int max_num_iterations_;
    double convergence_criterion_;
    int max_num_threads_;

   private:
    core::Matrix4dR align(const std::vector<core::Vector3d>& frame, const core::impl::DeviceVoxelMap& voxel_map,
                          const double max_distance, const double kernel_scale) const {
        core::Matrix4dR pose;
        ob_icp_io io{};
        io.source.dtype = OB_F64;
        io.source.points = frame.empty() ? nullptr : frame[0].data();
        io.source.n = frame.size();
        io.max_distance = max_distance;
        io.kernel_scale = kernel_scale;
        io.max_num_iterations = max_num_iterations_;
        io.convergence_criterion = convergence_criterion_;
        io.pose = pose.m.data();
        core::b200::check(ob_icp_align(voxel_map.handle(), &io, core::b200::thread_stream()));
        return pose;
    }
};

}  // namespace mapping
}  // namespace sdk
}  // namespace ouster
