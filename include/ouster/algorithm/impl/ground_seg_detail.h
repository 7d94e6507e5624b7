// ground_seg_detail.h -- impl::get_ground_mask (mirrors ouster_algorithm/src/ground_seg.cpp:1137-1343) over the
// C ABI's ob_ground_mask: one frame, or every frame of a set in one call (GroundSegEngine::update).
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/chanfield.h"
#include "ouster/core/lidar_frame.h"
#include "ouster/core/sensor_info.h"
#include "ouster/core/xyzlut.h"
#include "ouster_b200.h"

namespace ouster {
namespace sdk {
namespace algorithm {
namespace impl {

/// SensorInfo::num_returns of the reference: 2 for the dual-return lidar profiles, else 1.
inline int num_returns(const core::SensorInfo& info) {
    using P = core::UDPProfileLidar;
    switch (info.format.udp_profile_lidar) {
        case P::RNG19_RFL8_SIG16_NIR16_DUAL:
        case P::FUSA_RNG15_RFL8_NIR8_DUAL:
        case P::RNG15_RFL8_NIR8_DUAL:
        case P::RNG19_RFL8_SIG16_ZONE16_DUAL:
        case P::RNG19_RFL8_SIG16_NIR16_RGB16_DUAL:
            return 2;
        default:
            return 1;
    }
}

/// One frame as an ob_ground_item: its range images (RANGE, RANGE2, ... up to the first missing one, at most
/// num_returns), NORMALS / NORMALS2 when the frame has them as float32, else normals computed by the call.
struct GroundFrame {
    std::vector<const uint32_t*> ranges;
    std::vector<uint8_t*> masks;
    ob_ground_item item{};

    /// masks: at least as many h x w buffers as the frame has returns, else the reference's error
    GroundFrame(const core::LidarFrame& frame, const core::XYZLut& lut, const std::vector<uint8_t*>& out,
                size_t mask_h, size_t mask_w)
        : masks(out) {
        if (!frame.sensor_info) throw std::invalid_argument("frame.sensor_info is required for get_ground_mask");
        if (!frame.has_field(core::ChanField::RANGE))
            throw std::invalid_argument("frame must contain RANGE field for get_ground_mask");
        const int max_returns = num_returns(*frame.sensor_info);
        ranges.push_back(frame.field<uint32_t>(core::ChanField::RANGE).data());
        for (int ret = 1; ret < max_returns; ++ret) {
            const std::string name = core::ChanField::return_field_name(core::ChanField::RANGE, ret);
            if (!frame.has_field(name)) break;
            ranges.push_back(frame.field<uint32_t>(name).data());
        }
        auto float_normals = [&](const char* name) -> const float* {
            if (!frame.has_field(name) || frame.field(name).tag() != core::ChanFieldType::FLOAT32) return nullptr;
            return frame.field(name).template get<float>();
        };
        item.lut = lut.device_lut().get();
        item.h = frame.h;
        item.w = frame.w;
        item.range = ranges.data();
        item.n_returns = ranges.size();
        item.status = frame.status().data();
        item.poses = frame.body_to_world().template get<double>();
        item.normals = float_normals(core::ChanField::NORMALS);
        item.normals2 = item.normals ? float_normals(core::ChanField::NORMALS2) : nullptr;
        item.sensor_to_body = frame.sensor_info->sensor_to_body.data();
        item.compute_normals = item.normals ? 0 : 1;
        item.masks = masks.data();
        item.n_masks = masks.size();
        item.mask_h = mask_h;
        item.mask_w = mask_w;
    }
    GroundFrame(const GroundFrame&) = delete;
    GroundFrame& operator=(const GroundFrame&) = delete;
};

/// impl::get_ground_mask (ground_seg.cpp:1319-1343): one mask of h*w per return found (1 = ground).
/// Throws std::invalid_argument with the reference's texts.
inline std::vector<std::vector<uint8_t>> get_ground_mask(const core::LidarFrame& frame, double grid_size,
                                                         const core::XYZLut& xyz_lut) {
    if (!frame.sensor_info) throw std::invalid_argument("frame.sensor_info is required for get_ground_mask");
    if (!frame.has_field(core::ChanField::RANGE))
        throw std::invalid_argument("frame must contain RANGE field for get_ground_mask");
    std::vector<std::vector<uint8_t>> out(static_cast<size_t>(num_returns(*frame.sensor_info)),
                                          std::vector<uint8_t>(frame.h * frame.w, 0u));
    std::vector<uint8_t*> ptrs;
    for (auto& m : out) ptrs.push_back(m.data());
    GroundFrame g(frame, xyz_lut, ptrs, frame.h, frame.w);
    core::b200::check(ob_ground_mask(&g.item, 1, grid_size, OB_GROUND_FINAL, core::b200::thread_stream()));
    out.resize(g.ranges.size());
    return out;
}

}  // namespace impl
}  // namespace algorithm
}  // namespace sdk
}  // namespace ouster
