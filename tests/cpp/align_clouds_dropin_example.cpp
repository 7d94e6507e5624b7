// align_clouds_dropin_example.cpp -- user code written against ouster_algorithm's point-cloud align_clouds
// overloads, compiled against the replacement header and run on the GPU.  Prints "ALIGN CLOUDS DROPIN OK" when every
// check passes.  Built and run by tests/test_gpu_align_clouds.py.
#include <cmath>
#include <cstdio>
#include <cstdint>
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

// six boxes standing on a floor, their sides and the floor sampled at pseudo-random places, with their normals
static void scene(core::DenseArray<double>& p, core::DenseArray<double>& n) {
    uint32_t state = 12345u;
    auto u = [&state] {
        state = 1664525u * state + 1013904223u;
        return static_cast<double>(state) / 4294967296.0;
    };
    std::vector<double> pts, nrm;
    const double boxes[6][5] = {{2, 3, 1, 4, 2.5},    {-5, -3, 2, 3, 1.5}, {4, 7, -6, -5, 3},
                                {-2, -1, -7, -4, 2}, {6, 6.5, 3, 5, 2},   {-7, -6, -3, 1, 1.2}};
    for (const auto& b : boxes) {
        const double x0 = b[0], x1 = b[1], y0 = b[2], y1 = b[3], h = b[4];
        const double faces[4][6] = {{x0, y0, x1, y0, 0, -1}, {x1, y0, x1, y1, 1, 0}, {x1, y1, x0, y1, 0, 1},
                                    {x0, y1, x0, y0, -1, 0}};
        for (const auto& f : faces)
            for (int i = 0; i < 600; ++i) {
                const double s = u(), z = u() * h;
                pts.insert(pts.end(), {f[0] + (f[2] - f[0]) * s, f[1] + (f[3] - f[1]) * s, z});
                nrm.insert(nrm.end(), {f[4], f[5], 0.0});
            }
    }
    for (int i = 0; i < 4000; ++i) {
        const double x = u() * 18 - 9, y = u() * 18 - 9;
        pts.insert(pts.end(), {x, y, 0.0});
        nrm.insert(nrm.end(), {0.0, 0.0, 1.0});
    }
    p = core::DenseArray<double>(pts.size() / 3, 3);
    n = core::DenseArray<double>(pts.size() / 3, 3);
    for (size_t i = 0; i < pts.size(); ++i) {
        p(i) = pts[i];
        n(i) = nrm[i];
    }
}

int main() {
    core::DenseArray<double> target, tn;
    scene(target, tn);
    // source = truth^-1 * target: yaw 60 degrees, translation (1.0, -0.5, 0.2)
    const double yaw = 60.0 * M_PI / 180.0, c = std::cos(yaw), s = std::sin(yaw), t[3] = {1.0, -0.5, 0.2};
    core::DenseArray<double> source(target.rows(), 3), sn(target.rows(), 3);
    for (size_t i = 0; i < target.rows(); ++i) {
        const double d[3] = {target(i, 0) - t[0], target(i, 1) - t[1], target(i, 2) - t[2]};
        source(i, 0) = c * d[0] + s * d[1];
        source(i, 1) = -s * d[0] + c * d[1];
        source(i, 2) = d[2];
        sn(i, 0) = c * tn(i, 0) + s * tn(i, 1);
        sn(i, 1) = -s * tn(i, 0) + c * tn(i, 1);
        sn(i, 2) = tn(i, 2);
    }
    auto near_truth = [&](const core::Matrix4dR& p) {
        // within 0.5 degrees and 5 cm
        return std::fabs(p(0, 0) - c) < 0.0087 && std::fabs(p(1, 0) - s) < 0.0087 &&
               std::hypot(std::hypot(p(0, 3) - t[0], p(1, 3) - t[1]), p(2, 3) - t[2]) < 0.05;
    };
    double conf = -1.0;
    CHECK(near_truth(algorithm::align_clouds(source, target)));
    CHECK(near_truth(algorithm::align_clouds(source, target, conf)) && conf > 0.8 && conf <= 1.0);
    CHECK(near_truth(algorithm::align_clouds(source, sn, target, tn)));
    conf = -1.0;
    CHECK(near_truth(algorithm::align_clouds(source, sn, target, tn, conf)) && conf > 0.8 && conf <= 1.0);
    // fewer than 20 feature points: the guess back, confidence 0
    core::Matrix4dR guess = core::Matrix4dR::Identity();
    guess(0, 3) = 0.5;
    core::DenseArray<double> few(5, 3);
    for (size_t i = 0; i < 15; ++i) few(i) = static_cast<double>(i);
    const core::Matrix4dR back = algorithm::align_clouds(few, target, guess, conf);
    CHECK(back(0, 3) == 0.5 && back(0, 0) == 1.0 && conf == 0.0);
    core::DenseArray<double> four(5, 4);
    expect_invalid([&] { algorithm::align_clouds(four, target); }, "source_points must have shape (N, 3)");
    core::DenseArray<double> short_n(3, 3);
    expect_invalid([&] { algorithm::align_clouds(source, sn, target, short_n); },
                   "target_points and target_normals must have the same number of rows");
    std::printf("ALIGN CLOUDS DROPIN OK\n");
    return 0;
}
