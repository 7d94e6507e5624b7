// dropin_example.cpp -- compiles against the replacement headers exactly like code written for
// ouster_core (cf. examples/representations_example.cpp:38-54, 85-131 of the reference):
//   XYZLut lut(info); auto cloud = lut(scan); destagger<double>(info, x_image) ...
// and exercises ScanBatcher / LidarScan (deprecated spellings) end to end on the GPU.
// Prints "DROPIN OK" when every check passes.  Built and run by tests/test_gpu_cpp_dropin.py.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/frame_pipeline.h"
#include "ouster/core/lidar_scan.h"  // deprecated forwarding header
#include "ouster/algorithm/normals.h"
#include "ouster/core/pose_util.h"
#include "ouster/core/xyzlut.h"

using namespace ouster::sdk::core;

#define CHECK(cond)                                                        \
    do {                                                                   \
        if (!(cond)) {                                                     \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            std::exit(1);                                                  \
        }                                                                  \
    } while (0)

template <typename Ex, typename F>
static void expect_throw(F&& fn, const std::string& text) {
    try {
        fn();
    } catch (const Ex& e) {
        if (std::string(e.what()).find(text) == std::string::npos) {
            std::fprintf(stderr, "wrong message: '%s' (wanted '%s')\n", e.what(), text.c_str());
            std::exit(1);
        }
        return;
    }
    std::fprintf(stderr, "expected exception '%s'\n", text.c_str());
    std::exit(1);
}

int main() {
    // ---- config 1 plumbing: OS1-64 1024x64 default sensor (SensorInfo::from_default) ----
    auto info = SensorInfo::from_default(LidarMode{1024, 10});
    info->format.udp_profile_lidar = UDPProfileLidar::RNG19_RFL8_SIG16_NIR16;
    info->fw_rev = "v3.2.1";
    const size_t h = info->format.pixels_per_column, w = info->format.columns_per_frame;
    CHECK(h == 64 && w == 1024);

    LidarScan scan(info);  // deprecated alias of LidarFrame
    CHECK(scan.has_field(ChanField::RANGE) && scan.has_field(ChanField::WINDOW));
    std::mt19937 gen(42);
    auto range = scan.field<uint32_t>(ChanField::RANGE);
    for (size_t i = 0; i < range.size(); ++i) range(i) = (gen() & 1) ? 0u : 1u + gen() % 10000u;
    auto refl = scan.field<uint8_t>(ChanField::REFLECTIVITY);
    for (size_t i = 0; i < refl.size(); ++i) refl(i) = static_cast<uint8_t>(gen());
    for (size_t c = 0; c < w; ++c) {
        scan.status()[c] = 1;
        scan.measurement_id()[c] = static_cast<uint16_t>(c);
        scan.timestamp()[c] = 1000 + c;
    }
    for (size_t p = 0; p < w / 16; ++p) scan.packet_timestamp()[p] = 10 + p;
    scan.frame_id = 700;

    // ---- XYZLut + cartesian ----
    XYZLut lut(*info);                 // double, built on the GPU from the beam intrinsics
    XYZLutT<float> lutf(lut);          // converting constructor
    CHECK(lut.direction.rows() == h * w && lut.h == h && lut.w == w);
    PointCloudXYZd cloud = lut(scan);
    PointCloudXYZf cloudf = lutf(scan);
    PointCloudXYZd cloud2 = cartesian(scan, lut);  // deprecated free function
    CHECK(cloud == cloud2);
    for (size_t i = 0; i < h * w; ++i) {
        const uint32_t r = range(i);
        for (int k = 0; k < 3; ++k) {
            const double want = r == 0 ? 0.0 : r * lut.direction(i, k) + lut.offset(i, k);
            CHECK(cloud(i, k) == want);  // same two roundings as the reference loop
            const float wantf = r == 0 ? 0.0f : r * lutf.direction(i, k) + lutf.offset(i, k);
            CHECK(cloudf(i, k) == wantf);
        }
    }
    // doc formula spot check of the LUT (python/src/ouster/sdk/examples/reference.py:18-76)
    {
        const size_t u = 5, v = 100, i = u * w + v;
        const double n = info->beam_to_lidar_transform(0, 3);
        const double te = 2.0 * M_PI * (1.0 - double(v) / w);
        const double ta = -2.0 * M_PI * info->beam_azimuth_angles[u] / 360.0;
        const double phi = 2.0 * M_PI * info->beam_altitude_angles[u] / 360.0;
        const double r = 5000;
        const double x = (r - n) * std::cos(te + ta) * std::cos(phi) + n * std::cos(te);
        const double z = (r - n) * std::sin(phi);
        const double gx = r * lut.direction(i, 0) + lut.offset(i, 0);
        const double gz = r * lut.direction(i, 2) + lut.offset(i, 2);
        CHECK(std::fabs(gx - (-x) * 0.001) < 1e-9);  // lidar_to_sensor = diag(-1,-1,1), tz = 36.18
        CHECK(std::fabs(gz - (z + 36.18) * 0.001) < 1e-9);
    }

    // ---- destagger / stagger ----
    img_t<uint32_t> destag = destagger<uint32_t>(*info, range);
    for (size_t u = 0; u < h; ++u) {
        const int s = info->format.pixel_shift_by_row[u];
        for (size_t j = 0; j < w; ++j) CHECK(destag(u, (j + s) % w) == range(u, j));
    }
    {   // untyped Field form + timestamp mapping (tests/destagger_test.cpp:135-161)
        Field fd = destagger(*info, scan.field(ChanField::RANGE));
        CHECK(std::memcmp(fd.get(), destag.data(), h * w * 4) == 0);
        for (size_t u = 0; u < h; u += 7)
            for (size_t j = 0; j < w; j += 13) {
                const int s = info->format.pixel_shift_by_row[u];
                const size_t src_col = (j + w - static_cast<size_t>(s)) % w;
                CHECK(column_timestamp_at_destaggered_pixel(u, j, info->format.pixel_shift_by_row,
                                                            scan.timestamp()) == 1000 + src_col);
            }
    }
    img_t<uint32_t> back = stagger<uint32_t>(*info, destag);
    for (size_t i = 0; i < h * w; ++i) CHECK(back(i) == range(i));
    expect_throw<std::invalid_argument>(
        [&] { destagger<uint32_t>(ArrayRef<const uint32_t>(range), std::vector<int>(h - 1, 0)); },
        "image height does not match shifts size");
    // LEGACY lidar packets with the newer IMU / zone-monitor packets: rejected like the reference (parsing.cpp:480-490)
    expect_throw<std::runtime_error>(
        [&] {
            DataFormat bad = info->format;
            bad.udp_profile_lidar = UDPProfileLidar::LEGACY;
            bad.udp_profile_imu = UDPProfileIMU::ACCEL32_GYRO32_NMEA;
            PacketFormat pf_bad(bad);
        },
        "Mixing LEGACY lidar packets");
    expect_throw<std::invalid_argument>(
        [&] {
            img_t<uint32_t> small(h, w / 2);
            destagger<uint32_t>(*info, small);
        },
        "Image resolution must match SensorInfo.");
    expect_throw<std::invalid_argument>(
        [&] {
            img_t<uint32_t> small(h, w / 2);
            cartesian(ArrayRef<const uint32_t>(small), lut);
        },
        "unexpected image dimensions");

    // ---- dewarp: per-column poses (python/tests/test_pose_util.py:334-360 known answer) ----
    {
        MatrixX16R<double> poses(4, 16);
        const double pose[16] = {1, 0, 0, 1, 0, 1, 0, -2, 0, 0, 1, 3, 0, 0, 0, 1};
        for (int w2 = 0; w2 < 4; ++w2)
            for (int k = 0; k < 16; ++k) poses(w2, k) = pose[k];
        PointCloudXYZd pts(8, 3);
        for (int i = 0; i < 8; ++i) {
            pts(i, 0) = i - 3;
            pts(i, 1) = i + 1;
            pts(i, 2) = i + 2;
        }
        PointCloudXYZd dw = dewarp<double>(pts, poses);
        for (int i = 0; i < 8; ++i)
            CHECK(dw(i, 0) == pts(i, 0) + 1 && dw(i, 1) == pts(i, 1) - 2 && dw(i, 2) == pts(i, 2) + 3);
        PointCloudXYZd tr = transform<double>(pts, pose);
        CHECK(tr == dw);
        // one-pass form: projection and per-column pose in the same kernel
        MatrixX16R<double> col_poses(w, 16);
        for (size_t c = 0; c < w; ++c)
            for (int k = 0; k < 16; ++k) col_poses(c, k) = pose[k] + (k % 4 == 3 && k < 12 ? 0.001 * c : 0.0);
        auto range = scan.field<uint32_t>(ChanField::RANGE);
        PointCloudXYZd two_pass = dewarp<double>(lut(range), col_poses);
        PointCloudXYZd fused = dewarp<double>(lut, range, col_poses);
        CHECK(fused == two_pass);
        // dewarp(frame, lut, min, max): posed, range-filtered, compacted points of the valid columns
        LidarScan posed(scan);
        for (size_t c = 0; c < w; ++c) {
            mat4d m = mat4d::Identity();
            m(0, 3) = 0.5 * c;
            posed.set_column_pose(static_cast<int>(c), m);
            posed.status()[c] = (c % 7 == 3) ? 0u : 1u;
        }
        CHECK(posed.get_column_pose(2)(0, 3) == 1.0 && posed.get_first_valid_column() == 0);
        std::vector<uint32_t> cols;
        PointCloudXYZd world = dewarp<double>(posed, lut, 0.3, 50.0, &cols);
        PointCloudXYZd cloud = lut(range);
        size_t k = 0;
        for (size_t c = 0; c < w; ++c) {
            if (c % 7 == 3) continue;
            for (size_t r = 0; r < h; ++r) {
                const uint32_t rv = range(r, c);
                if (rv < 300 || rv > 50000) continue;
                CHECK(k < static_cast<size_t>(world.rows()) && cols[k] == c);
                CHECK(world(k, 0) == cloud(r * w + c, 0) + 0.5 * c && world(k, 1) == cloud(r * w + c, 1));
                ++k;
            }
        }
        CHECK(k == static_cast<size_t>(world.rows()) && k > 0);
        expect_throw<std::out_of_range>([&] { posed.set_column_pose(-1, mat4d::Identity()); },
                                        "Column index out of range");
        // dewarp(frame_set, xyzluts, ...): the frames of a set, an empty slot skipped, concatenated
        auto f0 = std::make_shared<LidarScan>(posed);
        auto f2 = std::make_shared<LidarScan>(posed);
        f2->status()[1] = 0;
        FrameSet set{f0, nullptr, f2};
        std::vector<XYZLut> luts{lut, lut, lut};
        std::vector<uint32_t> fidx;
        PointCloudXYZd set_pts = dewarp<double>(set, luts, 0.3, 50.0, &fidx);
        PointCloudXYZd second = dewarp<double>(*f2, lut, 0.3, 50.0);
        CHECK(set_pts.rows() == world.rows() + second.rows() && fidx.size() == static_cast<size_t>(set_pts.rows()));
        CHECK(std::memcmp(set_pts.data(), world.data(), sizeof(double) * 3 * world.rows()) == 0);
        CHECK(std::memcmp(set_pts.data() + 3 * world.rows(), second.data(), sizeof(double) * 3 * second.rows()) == 0);
        CHECK(fidx.front() == 0 && fidx.back() == 2);
        // a window the reference cannot convert to uint32 millimetres throws; 4294967.295 m keeps every range
        expect_throw<std::invalid_argument>([&] { dewarp<double>(posed, lut, 0.0, HUGE_VAL); }, "range window");
        expect_throw<std::invalid_argument>([&] { dewarp<double>(set, luts, -1.0, 50.0); }, "range window");
        CHECK(dewarp<double>(posed, lut, 0.0, 4294967.295).rows() >= world.rows());
    }

    // ---- surface normals on the destaggered cloud (ouster/algorithm/normals.h) ----
    {
        auto range = scan.field<uint32_t>(ChanField::RANGE);
        PointCloudXYZd cloud = lut(range);
        img_t<uint32_t> rd = destagger<uint32_t>(*info, range);
        PointCloudXYZd xd(h * w, 3);
        destagger_into<double>(cloud.data(), h, w, 3, info->format.pixel_shift_by_row, false, xd.data());
        DenseArray<double> origins(w, 3);
        auto n = ouster::sdk::algorithm::normals(ArrayRef<const double>(xd), ArrayRef<const uint32_t>(rd),
                                                 ArrayRef<const double>(origins));
        CHECK(n.rows() == h * w && n.cols() == 3);
        size_t unit = 0;
        for (size_t i = 0; i < h * w; ++i) {
            const double l2 = n(i, 0) * n(i, 0) + n(i, 1) * n(i, 1) + n(i, 2) * n(i, 2);
            CHECK(l2 == 0.0 || std::abs(l2 - 1.0) < 1e-9);
            unit += l2 > 0.5;
            if (rd.data()[i] == 0) CHECK(l2 == 0.0);
        }
        CHECK(unit > 0);
        expect_throw<std::runtime_error>(
            [&] { ouster::sdk::algorithm::normals(ArrayRef<const double>(xd), ArrayRef<const uint32_t>(rd),
                                                  ArrayRef<const double>(origins), 1, 0.0174, -1.0); },
            "normals: target_distance_m must be positive");
    }

    // ---- frame_to_packets -> ScanBatcher -> LidarScan round trip ----
    PacketFormat pf(*info);
    std::vector<Packet> packets = impl::frame_to_packets(scan, pf, 0, 0);
    CHECK(packets.size() == w / 16);
    {   // the same packets from the GPU encoder (set_block of every field + CRC64 in one launch)
        std::vector<Packet> dev_packets = impl::frame_to_packets_device(scan, pf, 0, 0);
        CHECK(dev_packets.size() == packets.size());
        for (size_t i = 0; i < packets.size(); ++i) CHECK(dev_packets[i].buf == packets[i].buf);
    }
    LidarScan out(info);
    ScanBatcher batcher(*info);  // deprecated alias of FrameBatcher
    for (size_t i = 0; i < packets.size(); ++i) {
        const bool done = batcher(packets[i], out);
        CHECK(done == (i + 1 == packets.size()));
    }
    CHECK(out.frame_id == 700);
    for (const auto& name : {ChanField::RANGE, ChanField::REFLECTIVITY}) CHECK(out.field(name) == scan.field(name));
    for (size_t c = 0; c < w; ++c) CHECK(out.timestamp()[c] == 1000 + c && out.status()[c] == 1);
    expect_throw<std::invalid_argument>(
        [&] {
            LidarScan wrong(32, 512, UDPProfileLidar::RNG19_RFL8_SIG16_NIR16, 16);
            batcher.batch(packets[0], wrong);
        },
        "unexpected frame dimensions");

    // ---- extension: FramePipeline keeps several frames in flight ----
    {
        FusedCloud proto;
        XYZLutT<float> flut(*info);
        proto.lut = flut.device_lut();
        proto.pixel_shift_by_row = info->format.pixel_shift_by_row;
        FramePipeline pipe(info, 2, &proto);
        size_t finished = 0;
        auto verify = [&](const FramePipeline::Slot* s, int64_t want_id) {
            CHECK(s->frame.frame_id == want_id);
            CHECK(s->frame.field(ChanField::RANGE) == scan.field(ChanField::RANGE));
            PointCloudXYZf want = flut(scan.field<uint32_t>(ChanField::RANGE));
            CHECK(std::memcmp(want.data(), s->cloud.xyz_f32(0), sizeof(float) * 3 * h * w) == 0);
            ++finished;
        };
        for (int k = 0; k < 5; ++k) {
            scan.frame_id = 800 + k;
            for (const Packet& p : impl::frame_to_packets(scan, pf, 0, 0))
                if (const FramePipeline::Slot* s = pipe.push(p)) verify(s, 800 + static_cast<int64_t>(finished));
        }
        while (const FramePipeline::Slot* s = pipe.drain()) verify(s, 800 + static_cast<int64_t>(finished));
        CHECK(finished == 5);
    }

    std::printf("DROPIN OK launches=%zu\n", batcher.gpu_launches());
    return 0;
}
