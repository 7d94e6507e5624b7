// image_dropin_example.cpp -- user code written against ouster_core's AutoExposure, BeamUniformityCorrector and
// LocalToneMapper, compiled against the replacement header and run on the GPU.
//   image_dropin_example <h> <w> <frames> <in.bin> <out.bin>
// in.bin: frames x (h x w float mono), frames x (h x w x 3 float rgb), frames x (h x w x 3 float16 rgb).
// Runs, frame by frame with update_state false on frame 2: AutoExposure on the mono frames, a
// BeamUniformityCorrector on them as double, AutoExposure on the rgb frames, and AutoExposure and LocalToneMapper on
// the float16 frames; writes the five results in that order to out.bin.  Prints "IMAGE DROPIN OK".
// Built and run by tests/test_gpu_image_dropin.py.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/image_processing.h"

using namespace ouster::sdk::core;
using namespace ouster::sdk::core::image;

#define CHECK(cond)                                                                      \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            std::exit(1);                                                                \
        }                                                                                \
    } while (0)

template <typename T>
static void put(std::ofstream& f, const T* p, size_t n) {
    f.write(reinterpret_cast<const char*>(p), std::streamsize(n * sizeof(T)));
}

int main(int argc, char** argv) {
    CHECK(argc == 6);
    const size_t h = std::strtoul(argv[1], nullptr, 10), w = std::strtoul(argv[2], nullptr, 10);
    const size_t frames = std::strtoul(argv[3], nullptr, 10);
    const size_t n = h * w;
    std::vector<float> mono(frames * n), rgb(frames * n * 3);
    std::vector<float16_t> half(frames * n * 3);
    std::ifstream in(argv[4], std::ios::binary);
    in.read(reinterpret_cast<char*>(mono.data()), std::streamsize(mono.size() * 4));
    in.read(reinterpret_cast<char*>(rgb.data()), std::streamsize(rgb.size() * 4));
    in.read(reinterpret_cast<char*>(half.data()), std::streamsize(half.size() * 2));
    CHECK(in.good());

    // the reference's argument checks are absent; this port rejects what it cannot define
    try {
        AutoExposure bad(1.5, 0.1, 1);
        CHECK(false);
    } catch (const std::invalid_argument& e) {
        CHECK(std::string(e.what()) == "lo_percentile and hi_percentile must be in [0, 1)");
    }

    AutoExposure ae, ae_rgb, ae_half;
    BeamUniformityCorrector buc;
    LocalToneMapper ltm;
    std::ofstream out(argv[5], std::ios::binary);
    std::vector<float> r_ae, r_rgb, r_half, r_ltm;
    std::vector<double> r_buc;
    for (size_t f = 0; f < frames; ++f) {
        const bool us = f != 2;
        img_t<float> a(h, w);
        img_t<double> d(h, w);
        for (size_t i = 0; i < n; ++i) {
            a.data()[i] = mono[f * n + i];
            d.data()[i] = double(mono[f * n + i]);
        }
        ae.update(a, us);  // Eigen::Ref<img_t<float>> in the reference
        buc.update(d, us);
        std::vector<float> c(rgb.begin() + long(f * n * 3), rgb.begin() + long((f + 1) * n * 3));
        ae_rgb.update(RgbImageRef<float>(c.data(), h, w), us);
        std::vector<float> o1(n * 3), o2(n * 3);
        const RgbImageRef<const float16_t> src(half.data() + f * n * 3, h, w);
        ae_half.update(src, RgbImageRef<float>(o1.data(), h, w), us);
        ltm.update(src, RgbImageRef<float>(o2.data(), h, w), us);
        r_ae.insert(r_ae.end(), a.data(), a.data() + n);
        r_buc.insert(r_buc.end(), d.data(), d.data() + n);
        r_rgb.insert(r_rgb.end(), c.begin(), c.end());
        r_half.insert(r_half.end(), o1.begin(), o1.end());
        r_ltm.insert(r_ltm.end(), o2.begin(), o2.end());
    }
    CHECK(ae.state().initialized == 1);
    std::vector<double> dark(h);
    CHECK(buc.state(dark.data(), h).dark_count_rows == h);
    put(out, r_ae.data(), r_ae.size());
    put(out, r_buc.data(), r_buc.size());
    put(out, r_rgb.data(), r_rgb.size());
    put(out, r_half.data(), r_half.size());
    put(out, r_ltm.data(), r_ltm.size());
    CHECK(out.good());
    std::printf("IMAGE DROPIN OK\n");
    return 0;
}
