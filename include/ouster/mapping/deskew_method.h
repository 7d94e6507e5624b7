// deskew_method.h -- per-column poses for the frames of a FrameSet before registration
// (mirrors ouster_mapping/include/ouster/mapping/deskew_method.h and ouster_mapping/src/deskew_method.cpp:26-71,
// 790-832).  ConstantVelocityDeskewMethod::update is one ob_frames_interp_pose call for the whole set.
// IMU packets are not decoded by this library, so InertialIntegrationImuDeskewMethod is not provided: the factory
// refuses "imu_deskew", and "auto" when a sensor reports IMU measurements (DESIGN 9).
#pragma once
#include <cstdint>
#include <deque>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/frame_set.h"
#include "ouster/core/lidar_frame.h"
#include "ouster/core/sensor_info.h"
#include "ouster/core/typedefs.h"

namespace ouster {
namespace sdk {
namespace mapping {

/// Base of the deskew methods: keeps the last two registered poses (deskew_method.h DeskewMethod).
class DeskewMethod {
   public:
    DeskewMethod(const std::vector<std::shared_ptr<core::SensorInfo>>& infos,
                 const core::Matrix4dR& initial_pose = core::Matrix4dR::Identity())
        : initial_pose_(initial_pose) {
        if (infos.empty()) throw std::invalid_argument("No sensor info provided for slam");
    }
    virtual ~DeskewMethod() = default;
    DeskewMethod(const DeskewMethod&) = delete;
    DeskewMethod& operator=(const DeskewMethod&) = delete;

    /// set the per-column poses (body_to_world) of the valid columns of every frame of the set
    virtual void update(core::FrameSet& frame_set) = 0;

    virtual void set_last_pose(int64_t timestamp_ns, const core::Matrix4dR& pose) {
        if (ts_list_.size() >= 2) {
            ts_list_.pop_front();
            pose_list_.pop_front();
        }
        ts_list_.push_back(timestamp_ns * 1e-9);
        pose_list_.push_back(pose);
    }

    virtual void finalize_after_registration(core::FrameSet& frame_set, int64_t anchor_timestamp_ns,
                                             const core::Matrix4dR& corrected_anchor_pose) {
        (void)frame_set;
        set_last_pose(anchor_timestamp_ns, corrected_anchor_pose);
    }

   protected:
    std::deque<double> ts_list_;
    std::deque<core::Matrix4dR> pose_list_;
    core::Matrix4dR initial_pose_;
};

/// Constant velocity between the last two poses (deskew_method.cpp:55-71): each valid column (status & 1) gets
/// the pose at its timestamp; before two poses are known, the initial pose.  Frames are written in slot order; a
/// decreasing valid timestamp throws std::invalid_argument ("x_interp values must be monotonically increasing:
/// ...") with the frames before it written.
class ConstantVelocityDeskewMethod : public DeskewMethod {
   public:
    using DeskewMethod::DeskewMethod;

    void update(core::FrameSet& frame_set) override {
        std::vector<ob_frame_poses_item> items(frame_set.size());
        for (size_t idx : frame_set.valid_indices()) {
            core::LidarFrame& f = *frame_set[idx];
            items[idx].timestamps = f.timestamp().data();
            items[idx].status = f.status().data();
            items[idx].poses = f.body_to_world().template get<double>();
            items[idx].w = f.w;
        }
        const bool init = ts_list_.size() < 2;
        core::b200::check(ob_frames_interp_pose(
            items.data(), items.size(), init ? 0.0 : ts_list_.front(),
            init ? initial_pose_.data() : pose_list_.front().data(), init ? 0.0 : ts_list_.back(),
            init ? nullptr : pose_list_.back().data(), nullptr, core::b200::thread_stream()));
    }
};

/// DeskewMethodFactory::create (deskew_method.cpp:790-832)
class DeskewMethodFactory {
   public:
    static std::unique_ptr<DeskewMethod> create(const std::string& method,
                                                const std::vector<std::shared_ptr<core::SensorInfo>>& infos,
                                                const core::Matrix4dR& initial_pose = core::Matrix4dR::Identity()) {
        bool has_imu_data = false;
        for (const auto& info : infos)
            if (info && info->format.imu_measurements_per_packet * info->format.imu_packets_per_frame > 0)
                has_imu_data = true;
        const char* imu_text = "IMU deskew is not supported: IMU packets are not decoded";
        if (method == "none") return nullptr;
        if (method == "constant_velocity") return std::make_unique<ConstantVelocityDeskewMethod>(infos, initial_pose);
        if (method == "imu_deskew") throw std::invalid_argument(imu_text);
        if (method == "auto") {
            if (has_imu_data) throw std::invalid_argument(imu_text);
            return std::make_unique<ConstantVelocityDeskewMethod>(infos, initial_pose);
        }
        throw std::invalid_argument("Invalid deskew_method: " + method);
    }
};

}  // namespace mapping
}  // namespace sdk
}  // namespace ouster
