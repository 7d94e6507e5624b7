// align_dropin_example.cpp -- user code written against ouster_algorithm's point_to_point_align and
// point_to_plane_align, the way the reference's tests call them, compiled against the replacement header and run on
// the GPU.  Prints "ALIGN DROPIN OK" when every check passes.  Built and run by tests/test_gpu_align_dropin.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/algorithm/align_clouds.h"

using namespace ouster::sdk;

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
    // python/tests/test_align_clouds.py: a 3x3x3 lattice moved by a translation
    core::DenseArray<double> source(27, 3), target(27, 3);
    const double t[3] = {0.1, -0.05, 0.025};
    int i = 0;
    for (double x : {-1.0, 0.0, 1.0})
        for (double y : {-1.0, 0.0, 1.0})
            for (double z : {-1.0, 0.0, 1.0}) {
                const double p[3] = {x, y, z};
                for (int d = 0; d < 3; ++d) {
                    source(i, d) = p[d];
                    target(i, d) = p[d] + t[d];
                }
                ++i;
            }
    const core::Matrix4dR pose = algorithm::point_to_point_align(source, target, core::Matrix4dR::Identity(), 0.5);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) CHECK(std::fabs(pose(r, c) - (r == c ? 1.0 : 0.0)) < 1e-10);
        CHECK(std::fabs(pose(r, 3) - t[r]) < 1e-10);
    }

    // a 5x5 plane lifted by 0.2 along its normal
    core::DenseArray<double> plane(25, 3), lifted(25, 3), normals(25, 3);
    i = 0;
    for (int x = 0; x < 5; ++x)
        for (int y = 0; y < 5; ++y, ++i) {
            plane(i, 0) = lifted(i, 0) = x;
            plane(i, 1) = lifted(i, 1) = y;
            plane(i, 2) = 0.0;
            lifted(i, 2) = 0.2;
            normals(i, 0) = normals(i, 1) = 0.0;
            normals(i, 2) = 1.0;
        }
    const core::Matrix4dR p2 = algorithm::point_to_plane_align(plane, lifted, normals, normals,
                                                               core::Matrix4dR::Identity(), 0.5);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) CHECK(std::fabs(p2(r, c) - (r == c ? 1.0 : 0.0)) < 1e-10);
    CHECK(std::fabs(p2(2, 3) - 0.2) < 1e-9 && std::fabs(p2(0, 3)) < 1e-9 && std::fabs(p2(1, 3)) < 1e-9);

    // defaults, and fewer than 20 rows give the initial guess back
    core::Matrix4dR guess = core::Matrix4dR::Identity();
    guess(0, 3) = 1.0 / 3.0;
    core::DenseArray<double> few(19, 3);
    for (size_t r = 0; r < 19; ++r)
        for (int d = 0; d < 3; ++d) few(r, d) = 0.1 * static_cast<double>(r + d);
    CHECK(algorithm::point_to_point_align(few, target, guess) == guess);
    CHECK(algorithm::point_to_point_align(source, target) == algorithm::point_to_point_align(source, target));

    // the reference's argument checks, in its order
    expect_invalid([&] { algorithm::point_to_point_align(source, target, guess, 0.0); },
                   "max_corr_dist must be finite and greater than zero");
    expect_invalid([&] { algorithm::point_to_plane_align(plane, lifted, normals, normals, guess, 0.5, 181.0); },
                   "max_normal_angle_deg must be finite and in [0, 180]");
    expect_invalid([&] { algorithm::point_to_plane_align(plane, lifted, few, normals); },
                   "source_points and source_normals must have the same number of rows");
    expect_invalid([&] { algorithm::point_to_plane_align(plane, lifted, normals, few); },
                   "target_points and target_normals must have the same number of rows");
    std::printf("ALIGN DROPIN OK\n");
    return 0;
}
