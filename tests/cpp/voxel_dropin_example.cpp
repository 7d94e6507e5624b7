// voxel_dropin_example.cpp -- user code written against the voxel-downsampling API of ouster_core /
// ouster_algorithm (core::voxel_downsample*, algorithm::voxel_downsample_with_normals), compiled against the
// replacement headers and run on the GPU.  Prints "VOXEL DROPIN OK" when every check passes.  Built and run by
// tests/test_gpu_voxel_dropin.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <set>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/algorithm/voxel_downsample.h"
#include "ouster/core/voxel_hash_map.h"

using namespace ouster::sdk;
using core::VoxelDownsampleStrategy;

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
    // python/tests/test_core.py:486-510, AVERAGE_POINT on points with two attribute columns
    const double f[4][5] = {{0, 1, 0, 10, 100}, {0, 1, 0, 12, 102}, {0, 2, 0, 20, 200}, {0, 2, 0, 22, 202}};
    core::DenseArray<double> frame(4, 5);
    for (size_t i = 0; i < 20; ++i) frame.data()[i] = f[i / 5][i % 5];
    auto one = core::voxel_downsample_xd(frame, 4.0, 1, 1, VoxelDownsampleStrategy::AVERAGE_POINT);
    CHECK(one.rows() == 1 && one.cols() == 5);
    CHECK(one(0, 1) == 1.5 && one(0, 3) == 16.0 && one(0, 4) == 151.0);
    auto two = core::voxel_downsample_xd(frame, 0.1, 1, 1, VoxelDownsampleStrategy::AVERAGE_POINT);
    CHECK(two.rows() == 2);
    CHECK(two(0, 1) + two(1, 1) == 3.0 && two(0, 3) + two(1, 3) == 32.0);

    // core::voxel_downsample: one representative per voxel, indices point at it, deterministic
    std::mt19937 gen(3);
    std::uniform_real_distribution<double> u(-5.0, 5.0);
    core::DenseArray<double> cloud(20000, 3);
    for (size_t i = 0; i < cloud.rows() * 3; ++i) cloud.data()[i] = u(gen);
    auto res = core::voxel_downsample(cloud, 1.0);
    const auto& pts = res.first;
    const auto& idx = res.second;
    CHECK(pts.rows() == idx.size() && pts.rows() > 900 && pts.rows() <= 1000);
    std::set<std::vector<int>> voxels;
    std::set<uint32_t> seen;
    for (size_t i = 0; i < pts.rows(); ++i) {
        CHECK(idx[i] < cloud.rows() && seen.insert(idx[i]).second);
        for (int k = 0; k < 3; ++k) CHECK(pts(i, k) == cloud(idx[i], k));
        CHECK(voxels.insert({int(std::floor(pts(i, 0))), int(std::floor(pts(i, 1))), int(std::floor(pts(i, 2)))}).second);
    }
    auto again = core::voxel_downsample(cloud, 1.0);
    CHECK(again.first == pts && again.second == idx);

    // voxel_downsample_3d defaults (1, 1, RANDOM): one point per voxel, taken from the input
    auto r3 = core::voxel_downsample_3d(cloud, 1.0);
    CHECK(r3.rows() == pts.rows());
    auto f3 = core::voxel_downsample_3d(cloud, 1.0, 4, 1, VoxelDownsampleStrategy::FIRST_N_POINT);
    CHECK(f3.rows() > r3.rows());

    // algorithm::voxel_downsample_with_normals
    core::DenseArray<double> p(3, 3), n(3, 3);
    const double pv[9] = {0.1, 0.1, 0.1, 0.3, 0.1, 0.1, 5.2, 0.0, 0.0};
    const double nv[9] = {0.0, 0.0, 2.0, 0.0, 3.0, 0.0, 1.0, 0.0, 0.0};
    for (int i = 0; i < 9; ++i) {
        p.data()[i] = pv[i];
        n.data()[i] = nv[i];
    }
    auto pn = algorithm::voxel_downsample_with_normals(p, n, 1.0);
    CHECK(pn.first.rows() == 2 && pn.second.rows() == 2);
    CHECK(pn.first(0, 0) == (0.1 + 0.3) / 2 && pn.first(1, 0) == 5.2);
    CHECK(std::fabs(pn.second(0, 1) - std::sqrt(0.5)) < 1e-15 && pn.second(1, 0) == 1.0);

    // the reference's exception texts, and an empty frame skipping every check
    expect_invalid([&] { core::voxel_downsample_3d(cloud, -1.0, 0); }, "max_points_per_voxel must be greater than 0");
    expect_invalid([&] { core::voxel_downsample_3d(cloud, 0.0); }, "voxel_size must be greater than 0");
    expect_invalid([&] { core::voxel_downsample_xd(core::DenseArray<double>(4, 2), 1.0); },
                   "voxel_downsample_xd: frame must have at least 3 columns");
    expect_invalid([&] { core::voxel_downsample_xd(frame, 1.0, 1, 1, static_cast<VoxelDownsampleStrategy>(7)); },
                   "voxel_downsample_xd: unknown strategy");
    expect_invalid([&] { algorithm::voxel_downsample_with_normals(frame, n, 1.0); },
                   "voxel_downsample_with_normals expects Nx3 inputs");
    expect_invalid([&] { algorithm::voxel_downsample_with_normals(cloud, n, 1.0); },
                   "voxel_downsample_with_normals points/normals size mismatch");
    expect_invalid([&] { algorithm::voxel_downsample_with_normals(p, n, 0.0); },
                   "voxel_downsample_with_normals voxel_size must be > 0");
    CHECK(core::voxel_downsample_xd(core::DenseArray<double>(0, 4), -1.0, 0).cols() == 4);
    CHECK(core::voxel_downsample(core::DenseArray<double>(0, 3), -1.0).second.empty());

    std::printf("VOXEL DROPIN OK (%zu of %zu points kept)\n", pts.rows(), cloud.rows());
    return 0;
}
