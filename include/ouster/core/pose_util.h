// pose_util.h -- per-column pose application to point clouds and pose interpolation
// (mirrors ouster_core/include/ouster/core/pose_util.h:24-160, 316-434; SURVEY 8f #1).  The loops run on the
// GPU (ob_dewarp, ob_interp_pose).
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <type_traits>
#include <vector>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/frame_set.h"
#include "ouster/core/lidar_frame.h"
#include "ouster/core/typedefs.h"
#include "ouster/core/xyzlut.h"

namespace ouster {
namespace sdk {
namespace core {

template <typename T>
using MatrixX16R = DenseArray<T>;  ///< W x 16: one flattened row-major 4x4 pose per row
using Poses = MatrixX16R<double>;

/// dewarp(dewarped, points, poses): dewarped[i*W + w] = R_w * points[i*W + w] + t_w
/// (pose_util.h:37-59).  points/dewarped are (H*W) x 3, poses W x 16.
template <typename T>
void dewarp(ArrayRef<T> dewarped, const ArrayRef<const T>& points, const ArrayRef<const T>& poses) {
    if (poses.cols() != 16 || points.cols() != 3 || dewarped.rows() != points.rows() ||
        poses.rows() == 0 || points.rows() % poses.rows() != 0)
        throw std::runtime_error("Number of points per set must match number of poses");
    b200::check(ob_dewarp(impl::lut_dtype<T>(), points.data(), poses.data(), points.rows(), poses.rows(),
                          dewarped.data(), b200::thread_stream()));
    b200::synchronize();
}

template <typename T>
PointCloudXYZ<T> dewarp(const PointCloudXYZ<T>& points, const MatrixX16R<T>& poses) {
    PointCloudXYZ<T> out(points.rows(), points.cols());
    dewarp<T>(ArrayRef<T>(out), ArrayRef<const T>(points), ArrayRef<const T>(poses));
    return out;
}

/// dewarp(lut, range, poses) == dewarp(lut(range), poses) in ONE pass over memory (extension:
/// the fusion the reference asks for in impl/dewarp_impl.h:27-29): point (row, col) of the staggered
/// cloud becomes R_col * p + t_col.  range is H x W, poses W x 16.
template <typename T>
PointCloudXYZ<T> dewarp(const XYZLutT<T>& lut, const ArrayRef<const uint32_t>& range,
                        const MatrixX16R<T>& poses) {
    const size_t n = static_cast<size_t>(lut.h) * lut.w;
    if (static_cast<size_t>(range.rows()) * range.cols() != n)
        throw std::invalid_argument("unexpected image dimensions");
    if (poses.cols() != 16 || static_cast<size_t>(poses.rows()) != lut.w)
        throw std::runtime_error("Number of points per set must match number of poses");
    PointCloudXYZ<T> out(n, 3);
    ob_cloud_io io{};
    io.n_frames = 1;
    io.n_returns = 1;
    io.range = range.data();
    io.xyz = out.data();
    io.poses = poses.data();
    b200::check(ob_scan_to_cloud(lut.device_lut().get(), nullptr, 0, &io, b200::thread_stream()));
    b200::synchronize();
    return out;
}

/// dewarp(lidar_frame, xyzlut, min_range, max_range) (pose_util.h:456-485, impl/dewarp_impl.h:22-76):
/// world-frame points of the first return, columns between the first and last valid one in order,
/// status == 0 columns skipped, min_range <= r <= max_range (metres), each point posed with its
/// column's body_to_world.  Returns an n x 3 array (the reference's std::vector<Eigen::Vector3<T>>
/// has the same memory layout).  One fused GPU pass (ob_dewarp_frame).  Optional per-point
/// provenance like impl::dewarp_impl: column index and column timestamp.
template <typename T>
PointCloudXYZ<T> dewarp(const LidarFrame& lidar_frame, const XYZLutT<T>& xyzlut, double min_range,
                        double max_range, std::vector<uint32_t>* col_idxs = nullptr,
                        std::vector<uint64_t>* timestamps_ns = nullptr) {
    auto range = lidar_frame.field<uint32_t>(ChanField::RANGE);
    const size_t n = static_cast<size_t>(xyzlut.h) * xyzlut.w;
    if (static_cast<size_t>(range.rows()) * range.cols() != n || lidar_frame.w != xyzlut.w)
        throw std::invalid_argument("unexpected image dimensions");
    PointCloudXYZ<T> all(n, 3);
    std::vector<uint32_t> ci(col_idxs ? n : 0);
    std::vector<uint64_t> ts(timestamps_ns ? n : 0);
    ob_dewarp_frame_io io{};
    io.range = range.data();
    io.poses = lidar_frame.body_to_world().template get<double>();
    io.status = lidar_frame.status().data();
    io.timestamps = lidar_frame.timestamp().data();
    io.min_range = min_range;
    io.max_range = max_range;
    io.points = all.data();
    io.col_idx = col_idxs ? ci.data() : nullptr;
    io.timestamps_out = timestamps_ns ? ts.data() : nullptr;
    io.capacity = n;
    size_t count = 0;
    b200::check(ob_dewarp_frame(xyzlut.device_lut().get(), &io, &count, b200::thread_stream()));
    PointCloudXYZ<T> out(count, 3);
    if (count) std::memcpy(out.data(), all.data(), count * 3 * sizeof(T));
    if (col_idxs) col_idxs->insert(col_idxs->end(), ci.begin(), ci.begin() + static_cast<std::ptrdiff_t>(count));
    if (timestamps_ns)
        timestamps_ns->insert(timestamps_ns->end(), ts.begin(), ts.begin() + static_cast<std::ptrdiff_t>(count));
    return out;
}

/// dewarp(frame_set, xyzluts, min_range, max_range) (pose_util.h:475, impl/dewarp_impl.h:84-117): the
/// dewarped points of every frame of the set, frame after frame, each frame with its own LUT.  One batched
/// GPU pass for the whole set (ob_dewarp_frames: one launch).  Optional per-point
/// provenance like impl::dewarp_impl: frame index, column index, column timestamp (appended).
template <typename T>
PointCloudXYZ<T> dewarp(const FrameSet& frame_set, const std::vector<XYZLutT<T>>& xyzluts, double min_range,
                        double max_range, std::vector<uint32_t>* frame_idxs = nullptr,
                        std::vector<uint32_t>* col_idxs = nullptr, std::vector<uint64_t>* timestamps_ns = nullptr) {
    if (frame_set.size() != xyzluts.size())
        throw std::invalid_argument("Number of frames and number of XYZLuts must be the same");
    std::vector<ob_dewarp_frames_io> ios(frame_set.size());
    size_t cap = 0;
    for (size_t idx : frame_set.valid_indices()) {
        const LidarFrame& f = *frame_set[idx];
        const XYZLutT<T>& lut = xyzluts[idx];
        auto range = f.field<uint32_t>(ChanField::RANGE);
        const size_t n = static_cast<size_t>(lut.h) * lut.w;
        if (static_cast<size_t>(range.rows()) * range.cols() != n || f.w != lut.w)
            throw std::invalid_argument("unexpected image dimensions");
        ios[idx].lut = lut.device_lut().get();
        ios[idx].range = range.data();
        ios[idx].poses = f.body_to_world().template get<double>();
        ios[idx].status = f.status().data();
        ios[idx].timestamps = f.timestamp().data();
        cap += n;
    }
    PointCloudXYZ<T> all(cap, 3);
    const bool prov = frame_idxs || col_idxs || timestamps_ns;
    std::vector<uint32_t> fi(frame_idxs ? cap : 0), ci(col_idxs ? cap : 0);
    std::vector<uint64_t> ts(timestamps_ns ? cap : 0);
    (void)prov;
    size_t count = 0;
    if (cap)
        b200::check(ob_dewarp_frames(ios.data(), ios.size(), min_range, max_range, all.data(), cap,
                                     frame_idxs ? fi.data() : nullptr, col_idxs ? ci.data() : nullptr,
                                     timestamps_ns ? ts.data() : nullptr, nullptr, &count, b200::thread_stream()));
    PointCloudXYZ<T> out(count, 3);
    if (count) std::memcpy(out.data(), all.data(), count * 3 * sizeof(T));
    const auto n = static_cast<std::ptrdiff_t>(count);
    if (frame_idxs) frame_idxs->insert(frame_idxs->end(), fi.begin(), fi.begin() + n);
    if (col_idxs) col_idxs->insert(col_idxs->end(), ci.begin(), ci.begin() + n);
    if (timestamps_ns) timestamps_ns->insert(timestamps_ns->end(), ts.begin(), ts.begin() + n);
    return out;
}

namespace impl {
static_assert(sizeof(Matrix4dR) == 16 * sizeof(double), "Matrix4dR must be 16 packed doubles");

template <typename T>
constexpr int interp_x_dtype() {
    static_assert(std::is_same<T, double>::value || std::is_same<T, int64_t>::value,
                  "interp_pose takes double or int64_t x values");
    return std::is_same<T, double>::value ? OB_POSE_X_F64 : OB_POSE_X_I64;
}

/// one ob_interp_pose call on host buffers; the reference's std::invalid_argument texts come through check()
template <typename T>
void interp_pose_into(const T* x, size_t n, const T* known, size_t m, const void* poses_known, int pose_dtype,
                      int two_pose, void* out) {
    // the reference's first check, made here too so that it holds before the thread's stream (a device) exists
    if (!two_pose && m < 2) throw std::invalid_argument("Not enough evaluation poses for interpolation");
    ob_interp_pose_io io{};
    io.x_interp = x;
    io.n = n;
    io.x_known = known;
    io.m = m;
    io.x_dtype = interp_x_dtype<T>();
    io.pose_dtype = pose_dtype;
    io.two_pose = two_pose;
    io.poses_known = poses_known;
    io.poses = out;
    b200::check(ob_interp_pose(&io, b200::thread_stream()));
}
}  // namespace impl

/// interp_pose(x_interp, t0, x0, t1, x1) (pose_util.h:316-326): a * exp((x - t0) / (t1 - t0) * log(a^-1 b)) for
/// every x, extrapolating outside [t0, t1].  T is double or int64_t.  Throws std::invalid_argument with the
/// reference's texts: "Cannot interpolate with zero duration between poses", "x_interp values must be
/// monotonically increasing: <x> < <previous x>".
template <typename T>
std::vector<Matrix4dR> interp_pose(const std::vector<T>& x_interp, T t0, const Matrix4dR& x0, T t1,
                                   const Matrix4dR& x1) {
    const T known[2] = {t0, t1};
    Matrix4dR poses[2] = {x0, x1};
    std::vector<Matrix4dR> result(x_interp.size());
    impl::interp_pose_into<T>(x_interp.data(), x_interp.size(), known, 2, poses, OB_F64, 1, result.data());
    return result;
}

/// interp_pose(x_interp, x_known, poses_known) (pose_util.h:360-377): segments between consecutive knots,
/// the values after the last knot on the last segment.  Adds "x_known and poses_known sizes are not matching",
/// "Not enough evaluation poses for interpolation" and "input x_known values are not monotonically increasing or
/// values repeated" to the texts above.
template <typename T>
std::vector<Matrix4dR> interp_pose(const std::vector<T>& x_interp, const std::vector<T>& x_known,
                                   const std::vector<Matrix4dR>& poses_known) {
    if (x_known.size() != poses_known.size())
        throw std::invalid_argument("x_known and poses_known sizes are not matching");
    std::vector<Matrix4dR> result(x_interp.size());
    impl::interp_pose_into<T>(x_interp.data(), x_interp.size(), x_known.data(), x_known.size(), poses_known.data(),
                              OB_F64, 0, result.data());
    return result;
}

/// interp_pose(x_interp, x_known, poses_known) on MatrixX16R rows (pose_util.h:408-434): Scalar float is the
/// binding's interp_pose_float (known poses widened to double, each result rounded once).
template <typename T, typename Scalar>
MatrixX16R<Scalar> interp_pose(const std::vector<T>& x_interp, const std::vector<T>& x_known,
                               const MatrixX16R<Scalar>& poses_known) {
    static_assert(std::is_same<Scalar, double>::value || std::is_same<Scalar, float>::value,
                  "poses are float or double");
    if (x_known.size() != poses_known.rows())
        throw std::invalid_argument("x_known and poses_known sizes are not matching");
    if (poses_known.cols() != 16) throw std::invalid_argument("poses_known must have 16 columns");
    MatrixX16R<Scalar> result(x_interp.size(), 16);
    impl::interp_pose_into<T>(x_interp.data(), x_interp.size(), x_known.data(), x_known.size(), poses_known.data(),
                              std::is_same<Scalar, double>::value ? OB_F64 : OB_F32, 0, result.data());
    return result;
}

/// transform(points, pose): one 4x4 pose (16 values, row-major) for every point (pose_util.h:118-160).
template <typename T>
PointCloudXYZ<T> transform(const PointCloudXYZ<T>& points, const T* pose16) {
    PointCloudXYZ<T> out(points.rows(), points.cols());
    if (points.rows() == 0) return out;
    b200::check(ob_dewarp(impl::lut_dtype<T>(), points.data(), pose16, points.rows(), 1, out.data(),
                          b200::thread_stream()));
    b200::synchronize();
    return out;
}

}  // namespace core
}  // namespace sdk
}  // namespace ouster
