// voxel_hash_map.h -- voxel-grid downsampling (mirrors the free functions of
// ouster_core/include/ouster/core/voxel_hash_map.h:685-711 and ouster_core/src/voxel_hash_map.cpp:262-393;
// SURVEY 8f #2).  Same names, defaults and exception texts; the work runs on the GPU (ob_voxel_downsample,
// ouster-sdk_b200/csrc/ob_voxel.cu).
//
// VoxelHashMap3d (voxel_hash_map.h:352-510, voxel_hash_map.cpp:14-247) is a concrete class here whose table lives in
// device memory (ob_voxel_map, ouster-sdk_b200/csrc/ob_voxel_map.cu); its pointcloud() / extracted rows list voxels
// in creation order (the reference: tsl::robin_map order, DESIGN 9).
//
// Not part of this replacement: the VoxelHashMap class template itself (the bucket and strategy types),
// VoxelHashMapXd, the averaging / point-normal / indexed maps and get_voxel_bucket.
//
// Differences a caller can see:
//  * the reference's std::vector<Eigen::Vector3d> / ArrayX3dR arguments are n x 3 (n x d) row-major
//    ArrayRef<const double> views, results are DenseArray<double> (as in pose_util.h);
//  * voxel_downsample_3d / _xd emit voxels in the order of their first input row; the reference emits them
//    in tsl::robin_map iteration order (DESIGN 9).  voxel_downsample's order and indices are the reference's.
#pragma once
#include <cfloat>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <tuple>
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

/// VoxelHashMap3d = VoxelHashMap<Vector3i, Vector3d, DefaultVoxelBucket, first_n_point> (voxel_hash_map.h:352-510),
/// held in device memory.  Calls run on the calling thread's stream (b200::thread_stream()); the ones that return
/// data to the host wait for it.  min_pts_threshold is stored and has no effect, as in the reference.
class VoxelHashMap3d {
   public:
    using point_type = Vector3d;

    /// voxel_hash_map.cpp:14-41; @throws std::invalid_argument with the reference's texts, in its order
    explicit VoxelHashMap3d(double voxel_size, double max_distance = 100.0, std::size_t max_points_per_voxel = 20,
                            std::size_t min_pts_threshold = 1, std::size_t num_attributes = 0)
        : max_points_per_voxel_(max_points_per_voxel), min_pts_threshold_(min_pts_threshold) {
        if (max_points_per_voxel == 0) throw std::invalid_argument("max_points_per_voxel must be greater than 0");
        if (voxel_size <= 0) throw std::invalid_argument("voxel_size must be greater than 0");
        if (max_distance <= 0) throw std::invalid_argument("max_distance must be greater than 0");
        if (num_attributes != 0) throw std::invalid_argument("num_attributes must be 0 for a fixed-size PointType");
        b200::check(ob_voxel_map_create(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold,
                                        b200::device(), &map_));
    }
    ~VoxelHashMap3d() { ob_voxel_map_destroy(map_); }
    VoxelHashMap3d(const VoxelHashMap3d&) = delete;
    VoxelHashMap3d& operator=(const VoxelHashMap3d&) = delete;
    VoxelHashMap3d(VoxelHashMap3d&& o) noexcept
        : map_(o.map_), max_points_per_voxel_(o.max_points_per_voxel_), min_pts_threshold_(o.min_pts_threshold_) {
        o.map_ = nullptr;
    }

    bool empty() const { return sizes().first == 0; }
    void clear() { b200::check(ob_voxel_map_clear(map_, b200::thread_stream())); }

    /// add_points (voxel_hash_map.cpp:101-107): the same map as inserting the points one at a time
    void add_points(const std::vector<Vector3d>& points) { add_rows(points.empty() ? nullptr : points[0].data(), points.size()); }
    /// add_points(Eigen::Ref<const ArrayXXdR>) (voxel_hash_map.h:399-411): n x 3
    void add_points(const ArrayRef<const double>& points) {
        if (points.cols() != 3) throw std::invalid_argument("VoxelHashMap::add_points received unexpected point dimension");
        add_rows(points.data(), points.rows());
    }
    /// update (voxel_hash_map.cpp:78-83)
    void update(const std::vector<Vector3d>& points, const Vector3d& position) {
        add_points(points);
        remove_voxels_far_from_location(position);
    }

    /// voxel_hash_map.cpp:109-125
    void remove_voxels_far_from_location(const Vector3d& origin) {
        ob_voxel_map_cull_io io{};
        io.origin = origin.data();
        b200::check(ob_voxel_map_remove_far(map_, &io, b200::thread_stream()));
    }
    /// voxel_hash_map.cpp:127-154: the erased voxels' points, n x 3
    DenseArray<double> extract_voxels_far_from_location(const Vector3d& origin) {
        DenseArray<double> out(sizes().second, 3);
        ob_voxel_map_cull_io io{};
        io.origin = origin.data();
        io.extracted = out.data();
        io.capacity = out.rows();
        size_t n = 0;
        io.n_extracted = &n;
        b200::check(ob_voxel_map_remove_far(map_, &io, b200::thread_stream()));
        return impl::first_rows(out, n);
    }

    /// voxel_hash_map.cpp:62-76
    DenseArray<double> pointcloud() const {
        DenseArray<double> out(sizes().second, 3);
        size_t n = 0;
        b200::check(ob_voxel_map_point_cloud(map_, out.data(), out.rows(), &n, b200::thread_stream()));
        return impl::first_rows(out, n);
    }
    /// voxel_hash_map.cpp:43-56
    std::vector<Vector3d> pointcloud_vector() const {
        const DenseArray<double> a = pointcloud();
        std::vector<Vector3d> out(a.rows());
        for (size_t i = 0; i < a.rows(); ++i) out[i] = Vector3d(a(i, 0), a(i, 1), a(i, 2));
        return out;
    }

    /// voxel_hash_map.cpp:194-247: (closest point, squared distance); ((0,0,0), max_distance_sq) when none qualifies
    std::tuple<Vector3d, double> get_closest_neighbor(const Vector3d& query,
                                                      double max_distance_sq = DBL_MAX) const {
        ob_voxel_query_io io{};
        io.queries.dtype = OB_F64;
        io.queries.points = query.data();
        io.queries.n = 1;
        io.max_distance_sq = max_distance_sq;
        Vector3d nb;
        double d2 = 0.0;
        io.neighbors = nb.data();
        io.distances_sq = &d2;
        b200::check(ob_voxel_map_closest_neighbors(map_, &io, b200::thread_stream()));
        b200::synchronize();
        return std::make_tuple(nb, d2);
    }

    std::size_t max_points_per_voxel() const { return max_points_per_voxel_; }
    std::size_t min_pts_threshold() const { return min_pts_threshold_; }
    /// the C-ABI handle (ob_icp_align, batched ob_voxel_map_closest_neighbors)
    ob_voxel_map* handle() const { return map_; }

   private:
    std::pair<size_t, size_t> sizes() const {
        size_t v = 0, p = 0;
        b200::check(ob_voxel_map_size(map_, &v, &p, b200::thread_stream()));
        return {v, p};
    }
    void add_rows(const double* p, size_t n) {
        if (n == 0) return;
        ob_point_rows r{};
        r.dtype = OB_F64;
        r.points = p;
        r.n = n;
        b200::check(ob_voxel_map_add_points(map_, &r, b200::thread_stream()));
        b200::synchronize();  // the rows are the caller's memory, staged in stream order
    }

    ob_voxel_map* map_ = nullptr;
    std::size_t max_points_per_voxel_, min_pts_threshold_;
};

}  // namespace core
}  // namespace sdk
}  // namespace ouster
