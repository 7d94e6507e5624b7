// align_clouds.h -- algorithm::point_to_point_align and point_to_plane_align (mirrors
// ouster_algorithm/include/ouster/algorithm/align_clouds.h:20-84 and ouster_algorithm/src/align_clouds.cpp:1590-1874;
// DESIGN f-7), and the six point-cloud overloads of algorithm::align_clouds (align_clouds.h:183-320,
// align_clouds.cpp:2601-2651; DESIGN f-14).  Same names, defaults and std::invalid_argument texts; the work runs on
// the GPU (ob_cloud_align, ouster-sdk_b200/csrc/ob_align.cu; ob_align_clouds, ob_align_clouds.cu).
//
// Eigen is absent (as in ouster/core/typedefs.h): the clouds are core::ArrayRef<const double> views of n x 3
// row-major rows in place of Eigen::Ref<const ArrayX3dR>, and the pose is the core::Matrix4dR stand-in.
//
// Differences a caller can see:
//  * the pose agrees with a CPU restatement of the reference to about 1e-12, not bit for bit: the GPU sums the correspondences in a
//    fixed tree rather than in sequence, and device sin / cos / acos are not host libm (DESIGN 9); the iteration
//    count, the correspondences and the "return initial_guess" cases are the reference's;
//  * align_clouds: the FFT's rounding differs from Eigen's kissfft, so a near-tie between yaw candidates can be decided
//    differently from the reference, and feature points follow the first-appearance voxel order (DESIGN 9);
//  * the align_clouds overloads for LidarFrame pairs and for a FrameSet are not provided yet.
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

namespace detail {
inline core::Matrix4dR align_clouds_impl(core::ArrayRef<const double> source_points,
                                         const core::ArrayRef<const double>* source_normals,
                                         core::ArrayRef<const double> target_points,
                                         const core::ArrayRef<const double>* target_normals,
                                         const core::Matrix4dR& initial_guess, double* confidence) {
    ob_align_clouds_io io{};  // ob_align_clouds checks the shapes, with the reference's texts
    io.source = ob_point_rows{OB_F64, source_points.data(), source_points.rows(), nullptr, 0};
    io.source_cols = source_points.rows() ? source_points.cols() : 3;
    io.target = ob_point_rows{OB_F64, target_points.data(), target_points.rows(), nullptr, 0};
    io.target_cols = target_points.rows() ? target_points.cols() : 3;
    if (source_normals) {
        io.source_normals = source_normals->data();
        io.source_normal_rows = source_normals->rows();
        io.source_normal_cols = source_normals->rows() ? source_normals->cols() : 3;
        io.target_normals = target_normals->data();
        io.target_normal_rows = target_normals->rows();
        io.target_normal_cols = target_normals->rows() ? target_normals->cols() : 3;
    }
    io.initial_guess = initial_guess.data();
    io.compute_confidence = confidence != nullptr;
    core::Matrix4dR pose;
    io.pose = pose.m.data();
    io.confidence = confidence;
    core::b200::check(ob_align_clouds(&io, core::b200::thread_stream()));
    return pose;
}
}  // namespace detail

/// align_clouds (align_clouds.h:183-219): source_to_target_transform between two gravity-aligned point clouds with
/// no usable initial guess: a 360 degree yaw search by BEV cross-correlation, three ICP passes and an overlap check.
/// @throws std::invalid_argument "source_points must have shape (N, 3)" (and the target's)
inline core::Matrix4dR align_clouds(core::ArrayRef<const double> source_points,
                                    core::ArrayRef<const double> target_points,
                                    const core::Matrix4dR& initial_guess = core::Matrix4dR::Identity()) {
    return detail::align_clouds_impl(source_points, nullptr, target_points, nullptr, initial_guess, nullptr);
}
/// As above; confidence: the share of points with an XY neighbour in the other cloud, in [0, 1].
inline core::Matrix4dR align_clouds(core::ArrayRef<const double> source_points,
                                    core::ArrayRef<const double> target_points, const core::Matrix4dR& initial_guess,
                                    double& confidence) {
    return detail::align_clouds_impl(source_points, nullptr, target_points, nullptr, initial_guess, &confidence);
}
inline core::Matrix4dR align_clouds(core::ArrayRef<const double> source_points,
                                    core::ArrayRef<const double> target_points, double& confidence) {
    return align_clouds(source_points, target_points, core::Matrix4dR::Identity(), confidence);
}
/// align_clouds with normals (align_clouds.h:221-320): point-to-plane ICP, and normal-weighted BEV grids.
/// @throws std::invalid_argument the shape texts, or "source_points and source_normals must have the same number of
///         rows" (and the target's)
inline core::Matrix4dR align_clouds(core::ArrayRef<const double> source_points,
                                    core::ArrayRef<const double> source_normals,
                                    core::ArrayRef<const double> target_points,
                                    core::ArrayRef<const double> target_normals,
                                    const core::Matrix4dR& initial_guess = core::Matrix4dR::Identity()) {
    return detail::align_clouds_impl(source_points, &source_normals, target_points, &target_normals, initial_guess,
                                     nullptr);
}
inline core::Matrix4dR align_clouds(core::ArrayRef<const double> source_points,
                                    core::ArrayRef<const double> source_normals,
                                    core::ArrayRef<const double> target_points,
                                    core::ArrayRef<const double> target_normals, double& confidence) {
    return detail::align_clouds_impl(source_points, &source_normals, target_points, &target_normals,
                                     core::Matrix4dR::Identity(), &confidence);
}
inline core::Matrix4dR align_clouds(core::ArrayRef<const double> source_points,
                                    core::ArrayRef<const double> source_normals,
                                    core::ArrayRef<const double> target_points,
                                    core::ArrayRef<const double> target_normals, const core::Matrix4dR& initial_guess,
                                    double& confidence) {
    return detail::align_clouds_impl(source_points, &source_normals, target_points, &target_normals, initial_guess,
                                     &confidence);
}

}  // namespace algorithm
}  // namespace sdk
}  // namespace ouster
