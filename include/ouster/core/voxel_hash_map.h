// voxel_hash_map.h -- voxel-grid downsampling (mirrors the free functions of
// ouster_core/include/ouster/core/voxel_hash_map.h:685-711 and ouster_core/src/voxel_hash_map.cpp:262-393;
// SURVEY 8f #2).  Same names, defaults and exception texts; the work runs on the GPU (ob_voxel_downsample,
// ouster-sdk_b200/csrc/ob_voxel.cu).
//
// VoxelHashMap3d and VoxelHashMapXd (voxel_hash_map.h:352-517, voxel_hash_map.cpp:14-247) are concrete classes here
// over one device-resident map (ob_voxel_map, ouster-sdk_b200/csrc/ob_voxel_map.cu); their pointcloud() / extracted
// rows list voxels in creation order (the reference: tsl::robin_map order, DESIGN 9).  VoxelHashMapXd's points are
// std::vector<double> (VectorXd here) of 3 + num_attributes values.
//
// Not part of this replacement: the VoxelHashMap class template itself (the bucket and strategy types),
// the averaging / point-normal / indexed maps and get_voxel_bucket.
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

using VectorXd = std::vector<double>;  ///< stand-in for Eigen::VectorXd (VoxelHashMapXd's points)

namespace impl {
/// What VoxelHashMap3d and VoxelHashMapXd share: the device map, the constructor's checks and every call that takes
/// or returns rows of point_cols() doubles.  Calls run on the calling thread's stream (b200::thread_stream()); the
/// ones that return data to the host wait for it.  min_pts_threshold is stored and has no effect, as in the reference.
class DeviceVoxelMap {
   public:
    /// voxel_hash_map.cpp:14-41; @throws std::invalid_argument with the reference's texts, in its order
    DeviceVoxelMap(double voxel_size, double max_distance, std::size_t max_points_per_voxel,
                   std::size_t min_pts_threshold, std::size_t num_attributes, bool fixed_size)
        : max_points_per_voxel_(max_points_per_voxel), min_pts_threshold_(min_pts_threshold), cols_(3 + num_attributes) {
        if (max_points_per_voxel == 0) throw std::invalid_argument("max_points_per_voxel must be greater than 0");
        if (voxel_size <= 0) throw std::invalid_argument("voxel_size must be greater than 0");
        if (max_distance <= 0) throw std::invalid_argument("max_distance must be greater than 0");
        if (fixed_size && num_attributes != 0)
            throw std::invalid_argument("num_attributes must be 0 for a fixed-size PointType");
        b200::check(ob_voxel_map_create_xd(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold,
                                           num_attributes, b200::device(), &map_));
    }
    ~DeviceVoxelMap() { ob_voxel_map_destroy(map_); }
    DeviceVoxelMap(const DeviceVoxelMap&) = delete;
    DeviceVoxelMap& operator=(const DeviceVoxelMap&) = delete;
    DeviceVoxelMap(DeviceVoxelMap&& o) noexcept
        : map_(o.map_), max_points_per_voxel_(o.max_points_per_voxel_), min_pts_threshold_(o.min_pts_threshold_),
          cols_(o.cols_) {
        o.map_ = nullptr;
    }

    bool empty() const { return sizes().first == 0; }
    void clear() { b200::check(ob_voxel_map_clear(map_, b200::thread_stream())); }

    /// add_points(Eigen::Ref<const ArrayXXdR>) (voxel_hash_map.h:399-411): n x point_cols()
    void add_points(const ArrayRef<const double>& points) {
        if (points.cols() != cols_) throw std::invalid_argument("VoxelHashMap::add_points received unexpected point dimension");
        add_rows(points.data(), points.rows());
    }

    /// voxel_hash_map.cpp:62-76: n x point_cols()
    DenseArray<double> pointcloud() const {
        DenseArray<double> out(sizes().second, cols_);
        size_t n = 0;
        b200::check(ob_voxel_map_point_cloud(map_, out.data(), out.rows(), &n, b200::thread_stream()));
        return first_rows(out, n);
    }

    /// VoxelHashMap::point_cols(): 3 + num_attributes
    std::size_t point_cols() const { return cols_; }
    std::size_t max_points_per_voxel() const { return max_points_per_voxel_; }
    std::size_t min_pts_threshold() const { return min_pts_threshold_; }
    /// the C-ABI handle (ob_icp_align, batched ob_voxel_map_closest_neighbors)
    ob_voxel_map* handle() const { return map_; }

   protected:
    std::pair<size_t, size_t> sizes() const {
        size_t v = 0, p = 0;
        b200::check(ob_voxel_map_size(map_, &v, &p, b200::thread_stream()));
        return {v, p};
    }
    void add_rows(const double* p, size_t n) {
        if (n == 0) return;
        ob_map_rows r{};
        r.rows = p;
        r.cols = cols_;
        r.n = n;
        b200::check(ob_voxel_map_add_rows(map_, &r, b200::thread_stream()));
        b200::synchronize();  // the rows are the caller's memory, staged in stream order
    }
    /// voxel_hash_map.cpp:109-125 (origin: x, y, z)
    void remove_far(const double* origin) {
        ob_voxel_map_cull_io io{};
        io.origin = origin;
        b200::check(ob_voxel_map_remove_far(map_, &io, b200::thread_stream()));
    }
    /// voxel_hash_map.cpp:127-154: the erased voxels' points, n x point_cols()
    DenseArray<double> extract_far(const double* origin) {
        DenseArray<double> out(sizes().second, cols_);
        ob_voxel_map_cull_io io{};
        io.origin = origin;
        io.extracted = out.data();
        io.capacity = out.rows();
        size_t n = 0;
        io.n_extracted = &n;
        b200::check(ob_voxel_map_remove_far(map_, &io, b200::thread_stream()));
        return first_rows(out, n);
    }
    /// voxel_hash_map.cpp:194-247 for the query x, y, z: the neighbour's point_cols() values into nb, the squared
    /// distance returned; zeros and max_distance_sq when nothing qualifies
    double closest(const double* query, double max_distance_sq, double* nb) const {
        ob_voxel_query_io io{};
        io.queries.dtype = OB_F64;
        io.queries.points = query;
        io.queries.n = 1;
        io.max_distance_sq = max_distance_sq;
        double d2 = 0.0;
        io.neighbors = nb;
        io.distances_sq = &d2;
        b200::check(ob_voxel_map_closest_neighbors(map_, &io, b200::thread_stream()));
        b200::synchronize();
        return d2;
    }

    ob_voxel_map* map_ = nullptr;
    std::size_t max_points_per_voxel_, min_pts_threshold_, cols_;
};
}  // namespace impl

/// VoxelHashMap3d = VoxelHashMap<Vector3i, Vector3d, DefaultVoxelBucket, first_n_point> (voxel_hash_map.h:352-510),
/// held in device memory.
class VoxelHashMap3d : public impl::DeviceVoxelMap {
   public:
    using point_type = Vector3d;

    /// voxel_hash_map.cpp:14-41; @throws std::invalid_argument with the reference's texts, in its order
    explicit VoxelHashMap3d(double voxel_size, double max_distance = 100.0, std::size_t max_points_per_voxel = 20,
                            std::size_t min_pts_threshold = 1, std::size_t num_attributes = 0)
        : DeviceVoxelMap(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold, num_attributes, true) {}

    using DeviceVoxelMap::add_points;
    /// add_points (voxel_hash_map.cpp:101-107): the same map as inserting the points one at a time
    void add_points(const std::vector<Vector3d>& points) { add_rows(points.empty() ? nullptr : points[0].data(), points.size()); }
    /// update (voxel_hash_map.cpp:78-83)
    void update(const std::vector<Vector3d>& points, const Vector3d& position) {
        add_points(points);
        remove_voxels_far_from_location(position);
    }

    /// voxel_hash_map.cpp:109-125
    void remove_voxels_far_from_location(const Vector3d& origin) { remove_far(origin.data()); }
    /// voxel_hash_map.cpp:127-154: the erased voxels' points, n x 3
    DenseArray<double> extract_voxels_far_from_location(const Vector3d& origin) { return extract_far(origin.data()); }

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
        Vector3d nb;
        const double d2 = closest(query.data(), max_distance_sq, nb.data());
        return std::make_tuple(nb, d2);
    }
};

/// VoxelHashMapXd = VoxelHashMap<Vector3i, VectorXd, DefaultVoxelBucket, first_n_point> (voxel_hash_map.h:512-513),
/// held in device memory: every point is x, y, z and num_attributes more values.  Voxels, the first_n_point gate, the
/// cull origin and the closest-neighbour query use x, y, z (impl::spatial_view); the attributes ride along.
class VoxelHashMapXd : public impl::DeviceVoxelMap {
   public:
    using point_type = VectorXd;

    /// voxel_hash_map.cpp:14-41; @throws std::invalid_argument with the reference's texts, in its order
    explicit VoxelHashMapXd(double voxel_size, double max_distance = 100.0, std::size_t max_points_per_voxel = 20,
                            std::size_t min_pts_threshold = 1, std::size_t num_attributes = 0)
        : DeviceVoxelMap(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold, num_attributes, false) {}

    using DeviceVoxelMap::add_points;
    /// add_points (voxel_hash_map.cpp:101-107); every point must have point_cols() values
    void add_points(const std::vector<VectorXd>& points) {
        std::vector<double> rows;
        rows.reserve(points.size() * point_cols());
        for (const VectorXd& p : points) {
            if (p.size() != point_cols())
                throw std::invalid_argument("VoxelHashMap::add_points received unexpected point dimension");
            rows.insert(rows.end(), p.begin(), p.end());
        }
        add_rows(rows.data(), points.size());
    }
    /// update (voxel_hash_map.cpp:78-83)
    void update(const std::vector<VectorXd>& points, const VectorXd& position) {
        add_points(points);
        remove_voxels_far_from_location(position);
    }

    /// voxel_hash_map.cpp:109-125 (the origin's x, y, z)
    void remove_voxels_far_from_location(const VectorXd& origin) { remove_far(spatial(origin)); }
    /// voxel_hash_map.cpp:127-154: the erased voxels' points, n x point_cols()
    DenseArray<double> extract_voxels_far_from_location(const VectorXd& origin) { return extract_far(spatial(origin)); }

    /// voxel_hash_map.cpp:43-56
    std::vector<VectorXd> pointcloud_vector() const {
        const DenseArray<double> a = pointcloud();
        std::vector<VectorXd> out(a.rows());
        for (size_t i = 0; i < a.rows(); ++i) out[i].assign(a.data() + i * a.cols(), a.data() + (i + 1) * a.cols());
        return out;
    }

    /// voxel_hash_map.cpp:170-247: (closest point with its attributes, squared distance); (point_cols() zeros,
    /// max_distance_sq) when none qualifies (PointDefaultValue::make(point_cols()))
    std::tuple<VectorXd, double> get_closest_neighbor(const VectorXd& query, double max_distance_sq = DBL_MAX) const {
        VectorXd nb(point_cols());
        const double d2 = closest(spatial(query), max_distance_sq, nb.data());
        return std::make_tuple(nb, d2);
    }

   private:
    static const double* spatial(const VectorXd& p) {
        if (p.size() < 3) throw std::invalid_argument("VoxelHashMap method expects a (3+attributes)-element point");
        return p.data();
    }
};

}  // namespace core
}  // namespace sdk
}  // namespace ouster
