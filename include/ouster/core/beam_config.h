// beam_config.h -- core::BeamConfig (mirrors ouster_core/include/ouster/core/beam_config.h and
// src/beam_config.cpp:14-52; DESIGN f-8): a sensor's beams and the two LUTs zones are rendered with.  The LUTs are
// built on the GPU in float64 with range unit 0.001 (ob_lut_from_intrinsics): `lut` from
// scale_translation(sensor_to_body) * lidar_to_sensor (present only with a sensor_to_body_transform), and
// `lut_no_sensor_to_body_transform` from lidar_to_sensor alone.  They are device tables (ob_lut handles) where the
// reference keeps host XYZLut objects.
#pragma once
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <vector>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/typedefs.h"
#include "ouster/core/zrb.h"

namespace ouster {
namespace sdk {
namespace core {

class BeamConfig {
   public:
    BeamConfig(uint32_t n_cols_init, const std::vector<double>& px_altitudes_init,
               const std::vector<double>& px_azimuths_init, const mat4d& beam_to_lidar_transform_init,
               const mat4d& lidar_to_sensor_transform_init, std::optional<mat4d> sensor_to_body_transform_init,
               float m_per_zmbin_init = DEFAULT_M_PER_ZMBIN, uint64_t serial_number_init = 0)
        : n_cols(n_cols_init),
          n_rows(static_cast<uint32_t>(px_altitudes_init.size())),
          beam_to_lidar_transform(beam_to_lidar_transform_init),
          lidar_to_sensor_transform(lidar_to_sensor_transform_init),
          sensor_to_body_transform(sensor_to_body_transform_init),
          m_per_zmbin(m_per_zmbin_init),
          serial_number(serial_number_init),
          px_altitudes(px_altitudes_init),
          px_azimuths(px_azimuths_init) {
        if (sensor_to_body_transform) {
            mat4d s2b = *sensor_to_body_transform;
            for (int r = 0; r < 3; ++r) s2b(r, 3) *= 1000;
            lut = make_lut(s2b * lidar_to_sensor_transform);
        }
        lut_no_sensor_to_body_transform = make_lut(lidar_to_sensor_transform);
        if (is_zero(beam_to_lidar_transform)) throw std::logic_error("BeamConfig: beam_to_lidar_transform not set");
        if (is_zero(lidar_to_sensor_transform))
            throw std::logic_error("BeamConfig: lidar_to_sensor_transform not set");
    }

    uint32_t n_cols;
    uint32_t n_rows;
    mat4d beam_to_lidar_transform;
    mat4d lidar_to_sensor_transform;
    std::optional<mat4d> sensor_to_body_transform;
    float m_per_zmbin;
    uint64_t serial_number;
    std::vector<double> px_altitudes;
    std::vector<double> px_azimuths;
    std::shared_ptr<ob_lut> lut;                              ///< with sensor_to_body; null without it
    std::shared_ptr<ob_lut> lut_no_sensor_to_body_transform;  ///< lidar_to_sensor only

   private:
    static bool is_zero(const mat4d& m) {
        for (double v : m.m)
            if (v != 0.0) return false;
        return true;
    }
    std::shared_ptr<ob_lut> make_lut(const mat4d& transform) const {
        ob_lut* h = nullptr;
        b200::check(ob_lut_from_intrinsics(OB_F64, n_cols, n_rows, 0.001, beam_to_lidar_transform.data(),
                                           transform.data(), px_azimuths.data(), px_azimuths.size(),
                                           px_altitudes.data(), px_altitudes.size(), b200::device(), &h));
        return std::shared_ptr<ob_lut>(h, [](ob_lut* p) { ob_lut_destroy(p); });
    }
};

}  // namespace core
}  // namespace sdk
}  // namespace ouster
