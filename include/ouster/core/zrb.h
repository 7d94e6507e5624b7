// zrb.h -- core::Zrb (mirrors ouster_core/include/ouster/core/zrb.h; DESIGN f-8): a rendered zone as near / far
// range images in mm and the transforms it was rendered with.  Reading and writing ZRB files (blob, save, hash)
// is not provided, and stl_hash stays unset.
#pragma once
#include <cstdint>
#include <optional>
#include <string>

#include "ouster/core/typedefs.h"

namespace ouster {
namespace sdk {
namespace core {

static constexpr float DEFAULT_M_PER_ZMBIN = 0.0074927621875f;

class Zrb {
   public:
    Zrb() = default;
    Zrb(uint32_t n_rows, uint32_t n_cols, float m_per_zmbin, uint64_t serial_number_init,
        const mat4d& beam_to_lidar, const mat4d& lidar_to_sensor, const mat4d& sensor_to_body)
        : near_range_mm(n_rows, n_cols),
          far_range_mm(n_rows, n_cols),
          serial_number(serial_number_init),
          beam_to_lidar_transform(beam_to_lidar),
          lidar_to_sensor_transform(lidar_to_sensor),
          sensor_to_body_transform(sensor_to_body),
          m_per_zmbin_(m_per_zmbin) {}

    float m_per_zmbin() const { return m_per_zmbin_; }

    img_t<uint32_t> near_range_mm;  ///< n_rows x n_cols, staggered, mm; 0 where the zone starts at the sensor
    img_t<uint32_t> far_range_mm;   ///< n_rows x n_cols, staggered, mm; 0 where no beam meets the zone
    uint64_t serial_number{0};
    mat4d beam_to_lidar_transform{mat4d::Identity()};
    mat4d lidar_to_sensor_transform{mat4d::Identity()};
    mat4d sensor_to_body_transform{mat4d::Identity()};
    std::optional<std::string> stl_hash;  ///< not computed here

    bool operator==(const Zrb& o) const {
        return near_range_mm == o.near_range_mm && far_range_mm == o.far_range_mm && serial_number == o.serial_number &&
               beam_to_lidar_transform == o.beam_to_lidar_transform &&
               lidar_to_sensor_transform == o.lidar_to_sensor_transform &&
               sensor_to_body_transform == o.sensor_to_body_transform && m_per_zmbin_ == o.m_per_zmbin_;
    }
    bool operator!=(const Zrb& o) const { return !(*this == o); }

   private:
    float m_per_zmbin_{DEFAULT_M_PER_ZMBIN};
};

}  // namespace core
}  // namespace sdk
}  // namespace ouster
