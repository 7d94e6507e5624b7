// voxel_map_xd_dropin_example.cpp -- user code written against ouster_core's VoxelHashMapXd and ouster_mapping's
// ICPRegistration::align_points_to_map(frame, VoxelHashMapXd, ...), the way the map exporter and
// python/tests/test_registration.py use them, compiled against the replacement headers and run on the GPU.  Prints
// "XD DROPIN OK" when every check passes.  Built and run by tests/test_gpu_voxel_map_xd.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "ouster/core/voxel_hash_map.h"
#include "ouster/mapping/icp_registration.h"

using namespace ouster::sdk;
using core::Vector3d;
using core::VectorXd;

#define CHECK(cond)                                                                      \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            std::exit(1);                                                                \
        }                                                                                \
    } while (0)

template <typename F>
static void expect_invalid(F&& fn, const std::string& text) {
    try {
        fn();
    } catch (const std::invalid_argument& e) {
        if (std::string(e.what()) != text) {
            std::fprintf(stderr, "wrong message: '%s' (wanted '%s')\n", e.what(), text.c_str());
            std::exit(1);
        }
        return;
    }
    std::fprintf(stderr, "expected std::invalid_argument '%s'\n", text.c_str());
    std::exit(1);
}

int main() {
    // voxel_hashmap_test.cpp:178-184
    expect_invalid([] { core::VoxelHashMap3d m(1.0, 100.0, 20, 1, 5); }, "num_attributes must be 0 for a fixed-size PointType");
    { core::VoxelHashMapXd m(1.0, 100.0, 20, 1, 5); CHECK(m.point_cols() == 8 && m.empty()); }

    // test_registration.py:49-70: a 4-point map with one attribute
    core::VoxelHashMapXd map(0.5, 10.0, 20, 1, 1);
    const double rows[4][4] = {{0, 0, 0, 10}, {1, 0, 0, 20}, {0, 1, 0, 30}, {0, 0, 1, 40}};
    map.add_points(core::ArrayRef<const double>(&rows[0][0], 4, 4));
    CHECK(!map.empty());
    const core::DenseArray<double> pc = map.pointcloud();
    CHECK(pc.rows() == 4 && pc.cols() == 4);
    for (size_t i = 0; i < 4; ++i)
        for (size_t j = 0; j < 4; ++j) CHECK(pc(i, j) == rows[i][j]);
    std::vector<Vector3d> frame;
    for (const auto& r : rows) frame.emplace_back(r[0] + 0.05, r[1] + 0.02, r[2] - 0.01);
    mapping::ICPRegistration reg(20);
    const core::Matrix4dR t = reg.align_points_to_map(frame, map, 0.5, 0.1);
    for (size_t i = 0; i < 4; ++i)
        for (int d = 0; d < 3; ++d) {
            const double v = t(d, 0) * frame[i][0] + t(d, 1) * frame[i][1] + t(d, 2) * frame[i][2] + t(d, 3);
            CHECK(std::fabs(v - rows[i][d]) < 0.05);
        }
    // the same x, y, z in a 3-d map: the same pose bit for bit
    core::VoxelHashMap3d map3(0.5, 10.0);
    std::vector<Vector3d> xyz;
    for (const auto& r : rows) xyz.emplace_back(r[0], r[1], r[2]);
    map3.add_points(xyz);
    const core::Matrix4dR t3 = reg.align_points_to_map(frame, map3, 0.5, 0.1);
    for (int i = 0; i < 16; ++i) CHECK(t.m[i] == t3.m[i]);

    // closest neighbour: the whole point; zeros and the bound when nothing qualifies
    VectorXd nb;
    double d2 = 0;
    std::tie(nb, d2) = map.get_closest_neighbor(VectorXd{0.9, 0.0, 0.0, 123.0});
    CHECK(nb.size() == 4 && nb[0] == 1.0 && nb[3] == 20.0 && std::fabs(d2 - 0.01) < 1e-12);
    std::tie(nb, d2) = map.get_closest_neighbor(VectorXd{9.0, 9.0, 9.0}, 2.0);
    CHECK(nb == VectorXd(4, 0.0) && d2 == 2.0);
    expect_invalid([&] { map.get_closest_neighbor(VectorXd{1.0, 2.0}); },
                   "VoxelHashMap method expects a (3+attributes)-element point");
    expect_invalid([&] { map.add_points(std::vector<VectorXd>{VectorXd{1, 2, 3}}); },
                   "VoxelHashMap::add_points received unexpected point dimension");

    // update = add + trim; extract carries the attributes
    map.update({VectorXd{50.0, 0.0, 0.0, 7.0}}, VectorXd{50.0, 0.0, 0.0});
    CHECK(map.pointcloud().rows() == 1);
    const core::DenseArray<double> ext = map.extract_voxels_far_from_location(VectorXd{-50.0, 0.0, 0.0, 0.0});
    CHECK(ext.rows() == 1 && ext(0, 0) == 50.0 && ext(0, 3) == 7.0 && map.empty());
    map.add_points(std::vector<VectorXd>{VectorXd{1, 2, 3, 4}});
    CHECK(map.pointcloud_vector().size() == 1 && map.pointcloud_vector()[0] == (VectorXd{1, 2, 3, 4}));
    map.clear();
    CHECK(map.empty());
    std::printf("XD DROPIN OK\n");
    return 0;
}
