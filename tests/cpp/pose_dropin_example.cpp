// pose_dropin_example.cpp -- plain g++ against include/ouster/core/pose_util.h and
// include/ouster/mapping/deskew_method.h: interp_pose in its three overloads (knot form, MatrixX16R<float>,
// two-pose form with int64_t x) on the reference's known answers, the reference's error texts, and
// ConstantVelocityDeskewMethod over a FrameSet.
//
//   pose_dropin_example host   argument checks that need no device (runs anywhere)
//   pose_dropin_example gpu    everything; prints "POSE <tag> <16 values>" lines for comparison with Python
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/pose_util.h"
#include "ouster/mapping/deskew_method.h"

using namespace ouster::sdk::core;
using ouster::sdk::mapping::ConstantVelocityDeskewMethod;
using ouster::sdk::mapping::DeskewMethodFactory;

#define CHECK(c)                                                         \
    do {                                                                 \
        if (!(c)) {                                                      \
            std::fprintf(stderr, "FAILED %s:%d %s\n", __FILE__, __LINE__, #c); \
            return 1;                                                    \
        }                                                                \
    } while (0)

template <typename F>
static std::string error_of(F&& fn) {
    try {
        fn();
    } catch (const std::invalid_argument& e) {
        return std::string("invalid_argument: ") + e.what();
    } catch (const std::exception& e) {
        return std::string("other: ") + e.what();
    }
    return "";
}

static Matrix4dR mat(const double* v) {
    Matrix4dR m;
    for (int k = 0; k < 16; ++k) m.m[k] = v[k];
    return m;
}

static void print_pose(const char* tag, const double* v) {
    std::printf("POSE %s", tag);
    for (int k = 0; k < 16; ++k) std::printf(" %.17g", v[k]);
    std::printf("\n");
}

// python/tests/test_pose_util.py:390-513, tests/interp_pose_test.cpp:50-140
static const double kCurr[16] = {0.950564, -0.29552, -0.0953745, 5, 0.294044, 0.955336, -0.0295028, 3,
                                 0.0998334, 0, 0.995004, 2, 0, 0, 0, 1};
static const double kNext[16] = {0.879923, -0.389418, -0.272192, 0, 0.372026, 0.921061, -0.115081, 0,
                                 0.29552, 0, 0.955336, 0, 0, 0, 0, 1};
static const double kExpected1[16] = {0.98756338, 0.149066, 0.04997893, -2.84746798, -0.14943741, 0.98876405,
                                      0.00375782, -0.91059756, -0.0488572, -0.01117981, 0.9987432, -0.7874577,
                                      0, 0, 0, 1};

int main(int argc, char** argv) {
    CHECK(argc == 2);
    const bool gpu = std::string(argv[1]) == "gpu";
    const std::vector<double> tss = {101000.0, 102000.0, 103000.0};
    const std::vector<Matrix4dR> poses = {Matrix4dR::Identity(), mat(kCurr), mat(kNext)};
    const std::vector<double> x = {100000.0, 100500.0, 101000.0, 101500.0, 102000.0, 102500.0, 103000.0, 103500.0};

    // argument checks the header and the C ABI make before any device work
    CHECK(error_of([&] { interp_pose(x, tss, std::vector<Matrix4dR>(2)); }) ==
          "invalid_argument: x_known and poses_known sizes are not matching");
    CHECK(error_of([&] { interp_pose(x, std::vector<double>{1.0}, std::vector<Matrix4dR>(1)); }) ==
          "invalid_argument: Not enough evaluation poses for interpolation");
    CHECK(error_of([&] { interp_pose(x, tss, MatrixX16R<float>(2, 16)); }) ==
          "invalid_argument: x_known and poses_known sizes are not matching");
    std::vector<std::shared_ptr<SensorInfo>> infos = {std::make_shared<SensorInfo>()};
    CHECK(error_of([&] { ConstantVelocityDeskewMethod m(std::vector<std::shared_ptr<SensorInfo>>{}); }) ==
          "invalid_argument: No sensor info provided for slam");
    CHECK(error_of([&] { DeskewMethodFactory::create("nope", infos); }) == "invalid_argument: Invalid deskew_method: nope");
    CHECK(error_of([&] { DeskewMethodFactory::create("imu_deskew", infos); }) ==
          "invalid_argument: IMU deskew is not supported: IMU packets are not decoded");
    CHECK(DeskewMethodFactory::create("none", infos) == nullptr);
    CHECK(DeskewMethodFactory::create("auto", infos) != nullptr);
    auto imu = std::make_shared<SensorInfo>();
    imu->format.imu_measurements_per_packet = 8;
    imu->format.imu_packets_per_frame = 16;
    CHECK(error_of([&] { DeskewMethodFactory::create("auto", {infos[0], imu}); }) ==
          "invalid_argument: IMU deskew is not supported: IMU packets are not decoded");
    if (!gpu) {
        std::printf("POSE DROPIN HOST OK\n");
        return 0;
    }

    // knot form: the reference's known answers (atol 1e-4)
    std::vector<Matrix4dR> got = interp_pose(x, tss, poses);
    CHECK(got.size() == 8);
    for (int k = 0; k < 16; ++k) CHECK(std::fabs(got[1].m[k] - kExpected1[k]) <= 1e-4);
    for (size_t i = 0; i < got.size(); ++i) print_pose(("knot" + std::to_string(i)).c_str(), got[i].data());
    // MatrixX16R<float>: interp_pose_float
    MatrixX16R<float> pk32(3, 16);
    for (size_t i = 0; i < 3; ++i)
        for (int k = 0; k < 16; ++k) pk32(i, k) = static_cast<float>(poses[i].m[k]);
    MatrixX16R<float> got32 = interp_pose(x, tss, pk32);
    for (size_t i = 0; i < got32.rows(); ++i) {
        double v[16];
        for (int k = 0; k < 16; ++k) v[k] = got32(i, k);
        print_pose(("f32_" + std::to_string(i)).c_str(), v);
    }
    // two-pose form, int64_t x
    const std::vector<int64_t> xi = {-500, 0, 250, 1000, 1500};
    std::vector<Matrix4dR> two = interp_pose<int64_t>(xi, 0, mat(kCurr), 1000, mat(kNext));
    for (size_t i = 0; i < two.size(); ++i) print_pose(("two" + std::to_string(i)).c_str(), two[i].data());
    // the reference's texts from the device checks
    const std::vector<double> unsorted = {100000.0, 100500.0, 101000.0, 102500.0, 102000.0, 101500.0, 103000.0,
                                          103500.0};
    CHECK(error_of([&] { interp_pose(unsorted, tss, poses); }) ==
          "invalid_argument: x_interp values must be monotonically increasing: 102000.000000 < 102500.000000");
    CHECK(error_of([&] { interp_pose(x, std::vector<double>{1.0, 3.0, 2.0}, poses); }) ==
          "invalid_argument: input x_known values are not monotonically increasing or values repeated");
    CHECK(error_of([&] { interp_pose<double>(x, 5.0, mat(kCurr), 5.0, mat(kNext)); }) ==
          "invalid_argument: Cannot interpolate with zero duration between poses");

    // ConstantVelocityDeskewMethod over a set with an empty slot: 64 columns, every third column invalid
    const size_t w = 64;
    FrameSet set({std::make_shared<LidarFrame>(4, w, UDPProfileLidar::RNG19_RFL8_SIG16_NIR16), nullptr,
                  std::make_shared<LidarFrame>(4, w, UDPProfileLidar::RNG19_RFL8_SIG16_NIR16)});
    for (size_t f : set.valid_indices()) {
        LidarFrame& fr = *set[f];
        for (size_t c = 0; c < w; ++c) {
            fr.timestamp().data()[c] = 1000000000ull + f * 100000000ull + c * 1000000ull;
            fr.status().data()[c] = c % 3 == 2 ? 0u : 1u;
        }
    }
    auto method = DeskewMethodFactory::create("constant_velocity", infos);
    method->update(set);  // no motion yet: the initial pose
    for (size_t c = 0; c < w; ++c)
        if (c % 3 != 2) CHECK(std::memcmp(set[0]->get_column_pose(static_cast<int>(c)).data(),
                                          Matrix4dR::Identity().data(), 128) == 0);
    method->set_last_pose(900000000, mat(kCurr));
    method->set_last_pose(1000000000, mat(kNext));
    method->update(set);
    for (size_t f : set.valid_indices())
        for (size_t c = 0; c < w; c += 5)
            print_pose(("deskew" + std::to_string(f) + "_" + std::to_string(c)).c_str(),
                       set[f]->get_column_pose(static_cast<int>(c)).data());
    std::printf("POSE DROPIN GPU OK\n");
    return 0;
}
