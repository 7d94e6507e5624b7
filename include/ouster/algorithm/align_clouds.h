// align_clouds.h -- algorithm::point_to_point_align and point_to_plane_align (mirrors
// ouster_algorithm/include/ouster/algorithm/align_clouds.h:20-84 and ouster_algorithm/src/align_clouds.cpp:1590-1874;
// DESIGN f-7).  Same names, defaults and std::invalid_argument texts; the ICP iterations run on the GPU
// (ob_cloud_align, ouster-sdk_b200/csrc/ob_align.cu).
//
// Eigen is absent (as in ouster/core/typedefs.h): the clouds are core::ArrayRef<const double> views of n x 3
// row-major rows in place of Eigen::Ref<const ArrayX3dR>, and the pose is the core::Matrix4dR stand-in.
//
// Differences a caller can see:
//  * the pose agrees with a CPU restatement of the reference to about 1e-12, not bit for bit: the GPU sums the correspondences in a
//    fixed tree rather than in sequence, and device sin / cos / acos are not host libm (DESIGN 9); the iteration
//    count, the correspondences and the "return initial_guess" cases are the reference's;
//  * the align_clouds(...) overloads (frame, FrameSet and point-cloud forms) are not provided.
#pragma once
#include <stdexcept>
#include <string>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/typedefs.h"

namespace ouster {
namespace sdk {
namespace algorithm {

namespace detail {
inline ob_point_rows align_rows(core::ArrayRef<const double> a, const char* name) {
    if (a.rows() && a.cols() != 3) throw std::invalid_argument(std::string(name) + " must be Nx3");
    ob_point_rows r{};
    r.dtype = OB_F64;
    r.points = a.data();
    r.n = a.rows();
    return r;
}
}  // namespace detail

/// point_to_point_align (align_clouds.h:20-46): source_to_target_transform by point-to-point ICP with MAD-scaled
/// Huber weights; initial_guess comes back when fewer than 20 usable points or correspondences exist.
/// @throws std::invalid_argument "max_corr_dist must be finite and greater than zero"
inline core::Matrix4dR point_to_point_align(core::ArrayRef<const double> source_points,
                                            core::ArrayRef<const double> target_points,
                                            const core::Matrix4dR& initial_guess = core::Matrix4dR::Identity(),
                                            double max_corr_dist = 0.25) {
    ob_cloud_align_io io{};
    io.mode = OB_ALIGN_POINT_TO_POINT;
    io.source = detail::align_rows(source_points, "source_points");
    io.target = detail::align_rows(target_points, "target_points");
    io.initial_guess = initial_guess.data();
    io.max_corr_dist = max_corr_dist;
    core::Matrix4dR pose;
    io.pose = pose.m.data();
    core::b200::check(ob_cloud_align(&io, core::b200::thread_stream()));
    return pose;
}

/// point_to_plane_align (align_clouds.h:48-84): source_to_target_transform by point-to-plane ICP; pairs whose
/// normals differ by more than max_normal_angle_deg are rejected, non-finite points and normals are ignored.
/// @throws std::invalid_argument "max_corr_dist must be finite and greater than zero",
///         "max_normal_angle_deg must be finite and in [0, 180]", or a "... must have the same number of rows" text
inline core::Matrix4dR point_to_plane_align(core::ArrayRef<const double> source_points,
                                            core::ArrayRef<const double> target_points,
                                            core::ArrayRef<const double> source_normals,
                                            core::ArrayRef<const double> target_normals,
                                            const core::Matrix4dR& initial_guess = core::Matrix4dR::Identity(),
                                            double max_corr_dist = 0.25, double max_normal_angle_deg = 20.0) {
    ob_cloud_align_io io{};
    io.mode = OB_ALIGN_POINT_TO_PLANE;
    io.source = detail::align_rows(source_points, "source_points");
    io.target = detail::align_rows(target_points, "target_points");
    io.source_normals = source_normals.data();
    io.source_normal_rows = source_normals.rows();
    io.target_normals = target_normals.data();
    io.target_normal_rows = target_normals.rows();
    io.initial_guess = initial_guess.data();
    io.max_corr_dist = max_corr_dist;
    io.max_normal_angle_deg = max_normal_angle_deg;
    core::Matrix4dR pose;
    io.pose = pose.m.data();
    core::b200::check(ob_cloud_align(&io, core::b200::thread_stream()));
    return pose;
}

}  // namespace algorithm
}  // namespace sdk
}  // namespace ouster
