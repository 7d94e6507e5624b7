// ground_dropin_example.cpp -- plain g++ against include/ouster/algorithm/ground_seg.h, written the reference's way:
// GroundSegEngine::create().update(frame_set), then read ChanField::GROUND.
//
//   ground_dropin_example host   the configuration check (runs anywhere)
//   ground_dropin_example gpu    a dual-return sensor over flat ground at 1.8 m: GROUND / GROUND2 added, an existing
//                                GROUND replaced, a stale GROUND2 removed, and impl::get_ground_mask agreeing
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/algorithm/ground_seg.h"

using namespace ouster::sdk::core;
using ouster::sdk::algorithm::GroundSegConfig;
using ouster::sdk::algorithm::GroundSegEngine;

#define CHECK(c)                                                                 \
    do {                                                                         \
        if (!(c)) {                                                              \
            std::fprintf(stderr, "FAILED %s:%d %s\n", __FILE__, __LINE__, #c); \
            return 1;                                                            \
        }                                                                        \
    } while (0)

static std::string error_of(double grid_size) {
    try {
        GroundSegConfig c;
        c.grid_size = grid_size;
        GroundSegEngine::create(c);
    } catch (const std::invalid_argument& e) {
        return e.what();
    }
    return "";
}

// a frame of a sensor 1.8 m above flat ground: every beam that points down hits it
static std::shared_ptr<LidarFrame> flat_frame(const std::shared_ptr<SensorInfo>& info, const XYZLut& lut, bool dual) {
    auto f = std::make_shared<LidarFrame>(info);
    auto rng = f->field<uint32_t>(ChanField::RANGE);
    for (size_t i = 0; i < f->h * f->w; ++i) {
        const double dz = lut.direction(i, 2) + 0.0;  // metres per millimetre
        const double r = dz < -1e-6 ? 1.8 / -dz : 0.0;
        rng.data()[i] = r > 0.0 && r < 60000.0 ? static_cast<uint32_t>(std::lround(r)) : 0u;
    }
    if (!dual && f->has_field(ChanField::RANGE2)) f->del_field(ChanField::RANGE2);
    if (dual) std::memcpy(f->field<uint32_t>(ChanField::RANGE2).data(), rng.data(), f->h * f->w * 4);
    for (size_t c = 0; c < f->w; ++c) f->status().data()[c] = 1u;
    return f;
}

int main(int argc, char** argv) {
    CHECK(argc == 2);
    CHECK(error_of(0.0) == "GroundSegConfig.grid_size must be > 0");
    CHECK(error_of(-1.0) == "GroundSegConfig.grid_size must be > 0");
    CHECK(error_of(NAN) == "GroundSegConfig.grid_size must be > 0");
    CHECK(error_of(0.5).empty());
    if (std::string(argv[1]) != "gpu") {
        std::printf("GROUND DROPIN HOST OK\n");
        return 0;
    }
    auto info = SensorInfo::from_default(LidarMode{1024, 10});
    info->format.udp_profile_lidar = UDPProfileLidar::RNG19_RFL8_SIG16_NIR16_DUAL;
    info->sn = 42;
    const XYZLut lut(*info, true);
    FrameSet set{flat_frame(info, lut, true), nullptr, flat_frame(info, lut, false)};
    // an existing GROUND is replaced, a stale GROUND2 on the single-return frame is removed
    set[0]->add_field(ChanField::GROUND, ChanFieldType::UINT8);
    std::memset(set[0]->field(ChanField::GROUND).get<uint8_t>(), 7, set[0]->h * set[0]->w);
    set[2]->add_field(ChanField::GROUND2, ChanFieldType::UINT8);

    auto ground = GroundSegEngine::create();
    ground->update(set);

    CHECK(set[0]->has_field(ChanField::GROUND) && set[0]->has_field(ChanField::GROUND2));
    CHECK(set[2]->has_field(ChanField::GROUND) && !set[2]->has_field(ChanField::GROUND2));
    for (size_t k : {size_t(0), size_t(2)}) {
        const LidarFrame& f = *set[k];
        const uint8_t* g = f.field(ChanField::GROUND).get<uint8_t>();
        const uint32_t* r = f.field<uint32_t>(ChanField::RANGE).data();
        size_t hits = 0, ground_px = 0;
        for (size_t i = 0; i < f.h * f.w; ++i) {
            CHECK(g[i] <= 1);
            hits += r[i] != 0;
            ground_px += g[i];
        }
        CHECK(hits > 1000 && ground_px >= hits * 99 / 100);
        const auto masks = ouster::sdk::algorithm::impl::get_ground_mask(f, 0.5, lut);
        CHECK(masks.size() == (k == 0 ? 2u : 1u));
        CHECK(std::memcmp(masks[0].data(), g, f.h * f.w) == 0);
        std::printf("GROUND frame %zu: %zu of %zu returns labelled ground\n", k, ground_px, hits);
    }
    std::printf("GROUND DROPIN GPU OK\n");
    return 0;
}
