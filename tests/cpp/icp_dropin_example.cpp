// icp_dropin_example.cpp -- user code written against ouster_core's VoxelHashMap3d and ouster_mapping's
// ICPRegistration / build_linear_system / AdaptiveThreshold, the way lio_slam.cpp uses them, compiled against the
// replacement headers and run on the GPU.  Prints "ICP DROPIN OK" when every check passes.  Built and run by
// tests/test_gpu_icp_dropin.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "ouster/core/voxel_hash_map.h"
#include "ouster/mapping/adaptive_threshold.h"
#include "ouster/mapping/icp_registration.h"

using namespace ouster::sdk;
using core::Vector3d;

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

// build_linear_system's leaf as icp_registration.cpp writes it: for up to 128 pairs the whole reduction is one leaf
static mapping::LinearSystem reference_leaf(const mapping::Correspondences& c, double ks) {
    mapping::LinearSystem ls;
    auto& jtj = ls.first;
    auto& jtr = ls.second;
    for (const auto& p : c) {
        const Vector3d& s = p.first;
        const double r[3] = {s[0] - p.second[0], s[1] - p.second[1], s[2] - p.second[2]};
        const double w = (ks * ks) / ((ks + ((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2])) *
                                      (ks + ((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2])));
        const double sx = s.x(), sy = s.y(), sz = s.z();
        const double wsx = w * sx, wsy = w * sy, wsz = w * sz;
        jtj(0, 0) += w;
        jtj(1, 1) += w;
        jtj(2, 2) += w;
        jtj(3, 1) -= wsz;
        jtj(3, 2) += wsy;
        jtj(4, 0) += wsz;
        jtj(4, 2) -= wsx;
        jtj(5, 0) -= wsy;
        jtj(5, 1) += wsx;
        const double wsx2 = wsx * sx, wsy2 = wsy * sy, wsz2 = wsz * sz;
        jtj(3, 3) += wsy2 + wsz2;
        jtj(4, 3) -= wsx * sy;
        jtj(4, 4) += wsx2 + wsz2;
        jtj(5, 3) -= wsx * sz;
        jtj(5, 4) -= wsy * sz;
        jtj(5, 5) += wsx2 + wsy2;
        const double cr[3] = {sy * r[2] - sz * r[1], sz * r[0] - sx * r[2], sx * r[1] - sy * r[0]};
        for (int k = 0; k < 3; ++k) {
            jtr(k) += w * r[k];
            jtr(3 + k) += w * cr[k];
        }
    }
    return ls;
}

int main() {
    // constructor checks, in the reference's order
    expect_invalid([] { core::VoxelHashMap3d m(0.5, 10.0, 0); }, "max_points_per_voxel must be greater than 0");
    expect_invalid([] { core::VoxelHashMap3d m(0.0, 10.0, 1); }, "voxel_size must be greater than 0");
    expect_invalid([] { core::VoxelHashMap3d m(0.5, -1.0, 1); }, "max_distance must be greater than 0");
    expect_invalid([] { core::VoxelHashMap3d m(0.5, 10.0, 20, 1, 2); }, "num_attributes must be 0 for a fixed-size PointType");

    // python/tests/test_registration.py: identity on an empty map, the shifted 4-point map recovered
    mapping::ICPRegistration reg(20);
    CHECK(reg.max_num_iterations_ == 20 && reg.convergence_criterion_ == 0.0001 && reg.max_num_threads_ > 0);
    core::VoxelHashMap3d map(0.5, 10.0);
    CHECK(map.empty() && map.max_points_per_voxel() == 20 && map.min_pts_threshold() == 1);
    const std::vector<Vector3d> pts = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    std::vector<Vector3d> shifted;
    for (const auto& p : pts) shifted.emplace_back(p[0] + 0.05, p[1] + 0.02, p[2] - 0.01);
    const core::Matrix4dR eye = reg.align_points_to_map(shifted, map, 1.0, 0.1);
    CHECK(eye == core::Matrix4dR::Identity());
    map.add_points(pts);
    CHECK(!map.empty() && map.pointcloud_vector() == pts);
    const core::Matrix4dR t = reg.align_points_to_map(shifted, map, 0.5, 0.1);
    for (size_t i = 0; i < pts.size(); ++i)
        for (int r = 0; r < 3; ++r) {
            const double v = t(r, 0) * shifted[i][0] + t(r, 1) * shifted[i][1] + t(r, 2) * shifted[i][2] + t(r, 3);
            CHECK(std::fabs(v - pts[i][r]) <= 0.05);
        }

    // get_closest_neighbor: exact match, bound prunes everything, sentinel
    Vector3d nb;
    double d2;
    std::tie(nb, d2) = map.get_closest_neighbor(Vector3d(1, 0, 0));
    CHECK(nb == Vector3d(1, 0, 0) && d2 == 0.0);
    std::tie(nb, d2) = map.get_closest_neighbor(Vector3d(0.3, 0, 0), 0.01);
    CHECK(nb == Vector3d(0, 0, 0) && d2 == 0.01);

    // build_linear_system: one leaf for <= 128 pairs, so the reference's own loop gives the same bits
    std::mt19937 gen(7);
    std::normal_distribution<double> nd(0.0, 3.0);
    mapping::Correspondences c;
    for (int i = 0; i < 100; ++i) {
        const Vector3d s(nd(gen), nd(gen), nd(gen));
        c.emplace_back(s, Vector3d(s[0] + nd(gen) * 0.01, s[1] - nd(gen) * 0.01, s[2] + nd(gen) * 0.02));
    }
    const mapping::LinearSystem got = mapping::build_linear_system(c, 0.3), want = reference_leaf(c, 0.3);
    CHECK(got.first.m == want.first.m && got.second.v == want.second.v);

    // update = add_points + remove_voxels_far_from_location; extraction returns the erased points
    core::VoxelHashMap3d m2(1.0, 2.0, 3);
    m2.update({{0.5, 0.5, 0.5}, {10.5, 0.5, 0.5}}, Vector3d(0, 0, 0));
    CHECK(m2.pointcloud_vector() == std::vector<Vector3d>({{0.5, 0.5, 0.5}}));
    m2.add_points(std::vector<Vector3d>({{-9.5, 0.5, 0.5}}));
    const auto ext = m2.extract_voxels_far_from_location(Vector3d(0, 0, 0));
    CHECK(ext.rows() == 1 && ext(0, 0) == -9.5);
    m2.clear();
    CHECK(m2.empty());

    // AdaptiveThreshold (python/tests/test_registration.py)
    mapping::AdaptiveThreshold th(100.0);
    CHECK(th.max_range_ == 100.0 && th.min_motion_threshold_ == 0.01 && th.compute_threshold() == 2.0);
    mapping::AdaptiveThreshold th2(100.0, 1.0);
    core::Matrix4dR dev = core::Matrix4dR::Identity();
    dev(0, 3) = 2.0;
    th2.update_model_deviation(dev);
    CHECK(th2.compute_threshold() > 1.0);
    std::printf("ICP DROPIN OK\n");
    return 0;
}
