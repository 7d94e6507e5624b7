// frame_ops_dropin_example.cpp -- user code written against ouster_core's frame_ops, compiled against the
// replacement header and run on the GPU.
//   frame_ops_dropin_example <h> <w> <in.bin> <out.bin>
// in.bin: RANGE u32 [h x w], SIGNAL u16 [h x w], F32 float [h x w], mask u8 [h x w], pixel_shift_by_row i32 [h].
// Runs on one frame: clip(RANGE, 100, 30000, 7), filter_field(SIGNAL, 1000, 20000, 1.7) on every pixel field,
// filter_uv("v", w / 4, w / 2, 9), mask; writes RANGE, SIGNAL, F32.  Then select_by_index({h - 1, 0, h / 2}) with
// and without metadata; writes the selected RANGE and the column field, checks the metadata and the reference's
// error texts.  Prints "FRAME OPS DROPIN OK".  Built and run by tests/test_gpu_frame_ops_dropin.py.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/frame_ops.h"

using namespace ouster::sdk::core;

#define CHECK(cond)                                                                      \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            std::exit(1);                                                                \
        }                                                                                \
    } while (0)

template <typename T>
static void get(std::ifstream& f, T* p, size_t n) {
    f.read(reinterpret_cast<char*>(p), static_cast<std::streamsize>(n * sizeof(T)));
}
template <typename T>
static void put(std::ofstream& f, const T* p, size_t n) {
    f.write(reinterpret_cast<const char*>(p), static_cast<std::streamsize>(n * sizeof(T)));
}

template <typename F>
static std::string error_of(F&& fn) {
    try {
        fn();
    } catch (const std::exception& e) {
        return e.what();
    }
    return "";
}

int main(int argc, char** argv) {
    CHECK(argc == 5);
    const size_t h = std::strtoul(argv[1], nullptr, 10), w = std::strtoul(argv[2], nullptr, 10), n = h * w;
    LidarFrameFieldTypes types = {FieldType("RANGE", ChanFieldType::UINT32), FieldType("SIGNAL", ChanFieldType::UINT16),
                                  FieldType("F32", ChanFieldType::FLOAT32),
                                  FieldType("COL", ChanFieldType::UINT32, {}, FieldClass::COLUMN_FIELD)};
    LidarFrame frame(h, w, types, 16);
    auto info = std::make_shared<SensorInfo>();
    info->prod_line = "OS-1-128";
    info->format.pixels_per_column = static_cast<uint32_t>(h);
    info->format.columns_per_frame = static_cast<uint32_t>(w);
    info->format.columns_per_packet = 16;
    info->beam_azimuth_angles.assign(h, 0.0);
    info->beam_altitude_angles.assign(h, 0.0);
    std::vector<uint8_t> m(n);
    std::vector<int32_t> shifts(h);
    {
        std::ifstream in(argv[3], std::ios::binary);
        CHECK(in.good());
        get(in, frame.field<uint32_t>("RANGE").data(), n);
        get(in, frame.field<uint16_t>("SIGNAL").data(), n);
        get(in, frame.field<float>("F32").data(), n);
        get(in, m.data(), n);
        get(in, shifts.data(), h);
        CHECK(in.good());
    }
    info->format.pixel_shift_by_row.assign(shifts.begin(), shifts.end());
    frame.sensor_info = info;
    uint32_t* col = static_cast<uint32_t*>(frame.field("COL").get());
    for (size_t c = 0; c < w; ++c) col[c] = static_cast<uint32_t>(c * 3 + 1);
    frame.frame_id = 42;

    frame_ops::clip(frame, {"RANGE"}, 100, 30000, 7);
    frame_ops::filter_field(frame, "SIGNAL", 1000, 20000, 1.7);
    frame_ops::filter_uv(frame, "v", w / 4, w / 2, 9);
    frame_ops::mask(frame, {}, ArrayRef<const uint8_t>(m.data(), h, w));

    std::ofstream out(argv[4], std::ios::binary);
    put(out, frame.field<uint32_t>("RANGE").data(), n);
    put(out, frame.field<uint16_t>("SIGNAL").data(), n);
    put(out, frame.field<float>("F32").data(), n);

    const std::vector<size_t> idx = {h - 1, 0, h / 2};
    LidarFrame plain = frame_ops::select_by_index(frame, idx);
    LidarFrame meta = frame_ops::select_by_index(frame, idx, true);
    CHECK(!plain.sensor_info && meta.sensor_info);
    CHECK(plain.h == 3 && plain.w == w && plain.frame_id == 42);
    CHECK(meta.sensor_info->prod_line == "OS-1-3" && meta.sensor_info->format.pixels_per_column == 3);
    CHECK(meta.sensor_info->format.pixel_shift_by_row[0] == shifts[h - 1]);
    CHECK(std::memcmp(plain.field("COL").get(), frame.field("COL").get(), w * 4) == 0);
    put(out, plain.field<uint32_t>("RANGE").data(), 3 * w);
    CHECK(frame_ops::reduce_by_factor_metadata(*info, h).h() == 1);
    CHECK(ProductInfo::create_product_info("OS-0-128-U1").beam_count == 128);

    const std::vector<std::string> col_only = {"COL"};
    std::printf("%s\n", error_of([&] { frame_ops::clip(frame, col_only, 0, 1); }).c_str());
    std::printf("%s\n", error_of([&] { frame_ops::filter_field(frame, "NOPE", 0, 1); }).c_str());
    std::printf("%s\n", error_of([&] { frame_ops::filter_uv(frame, "x", 0, 1); }).c_str());
    std::printf("%s\n", error_of([&] { frame_ops::clip(frame, {"RANGE"}, 0, 1, -1); }).c_str());
    std::printf("%s\n", error_of([&] { frame_ops::select_by_index(frame, {0, 0}); }).c_str());
    std::printf("%s\n", error_of([&] { frame_ops::reduce_factor_to_indices(3, 8); }).c_str());
    std::printf("FRAME OPS DROPIN OK\n");
    return 0;
}
