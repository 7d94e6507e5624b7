// ground_seg.h -- GroundSegConfig / GroundSegEngine (mirrors ouster_algorithm/include/ouster/algorithm/
// ground_seg.h and ground_seg.cpp:1346-1416).  update() segments every frame of a FrameSet in one
// ob_ground_mask call and writes the GROUND, GROUND2, ... pixel fields (uint8, 1 = ground).
#pragma once
#include <cmath>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <unordered_map>
#include <vector>

#include "ouster/algorithm/impl/ground_seg_detail.h"
#include "ouster/core/frame_set.h"

namespace ouster {
namespace sdk {
namespace algorithm {

struct GroundSegConfig {
    double grid_size = 0.5;  ///< Grid cell size in metres of the 2.5-D height map
};

class GroundSegEngine {
   public:
    virtual ~GroundSegEngine() = default;
    /// throws std::invalid_argument("GroundSegConfig.grid_size must be > 0") for a grid size that is not
    /// finite and positive
    static std::unique_ptr<GroundSegEngine> create(const GroundSegConfig& config = {});
    /// GROUND (and GROUND2, ... up to the sensor's returns) on every frame of the set: the fields are deleted and
    /// re-added zeroed, then filled; those beyond the returns a frame has (the first missing RANGEk) are removed.
    virtual void update(core::FrameSet& frames) = 0;
};

namespace impl {

class EnvelopeGridGroundSegEngine : public GroundSegEngine {
   public:
    explicit EnvelopeGridGroundSegEngine(const GroundSegConfig& config) : config_(config) {}

    void update(core::FrameSet& frames) override {
        std::vector<std::unique_ptr<GroundFrame>> held(frames.size());
        std::vector<ob_ground_item> items(frames.size());  // lut == NULL: an empty slot
        std::vector<std::pair<size_t, int>> max_returns;
        for (size_t idx : frames.valid_indices()) {
            auto& frame_ptr = frames[idx];
            if (!frame_ptr) continue;
            core::LidarFrame& frame = *frame_ptr;
            if (!frame.sensor_info)
                throw std::invalid_argument("frame.sensor_info is required for get_ground_mask");
            const core::XYZLut& lut = lut_of(*frame.sensor_info);
            const int n = num_returns(*frame.sensor_info);
            std::vector<uint8_t*> masks;
            for (int ret = 0; ret < n; ++ret) {
                const std::string name = core::ChanField::return_field_name(core::ChanField::GROUND, ret);
                if (frame.has_field(name)) frame.del_field(name);
                frame.add_field(name, core::ChanFieldType::UINT8, {}, core::FieldClass::PIXEL_FIELD);
                masks.push_back(frame.field(name).template get<uint8_t>());
            }
            held[idx] = std::make_unique<GroundFrame>(frame, lut, masks, frame.h, frame.w);
            items[idx] = held[idx]->item;
            max_returns.emplace_back(idx, n);
        }
        core::b200::check(ob_ground_mask(items.data(), items.size(), config_.grid_size, OB_GROUND_FINAL,
                                         core::b200::thread_stream()));
        // remove the GROUND fields of returns the frame does not have
        for (const auto& [idx, n] : max_returns) {
            core::LidarFrame& frame = *frames[idx];
            for (int ret = static_cast<int>(held[idx]->ranges.size()); ret < n; ++ret) {
                const std::string name = core::ChanField::return_field_name(core::ChanField::GROUND, ret);
                if (frame.has_field(name)) frame.del_field(name);
            }
        }
    }

   private:
    GroundSegConfig config_;
    std::unordered_map<uint64_t, core::XYZLut> luts_;  // one LUT per sensor serial number, as the reference

    const core::XYZLut& lut_of(const core::SensorInfo& info) {
        auto it = luts_.find(info.sn);
        if (it == luts_.end()) it = luts_.emplace(info.sn, core::XYZLut(info, true)).first;
        return it->second;
    }
};

}  // namespace impl

inline std::unique_ptr<GroundSegEngine> GroundSegEngine::create(const GroundSegConfig& config) {
    if (!std::isfinite(config.grid_size) || config.grid_size <= 0.0)
        throw std::invalid_argument("GroundSegConfig.grid_size must be > 0");
    return std::make_unique<impl::EnvelopeGridGroundSegEngine>(config);
}

}  // namespace algorithm
}  // namespace sdk
}  // namespace ouster
