// zone_state.h -- core::ZoneState (mirrors ouster_core/include/ouster/core/zone_state.h; DESIGN f-8): the packed
// 37-byte record a zone monitor reports per live zone, laid out as ob_zone_state.
#pragma once
#include <cstdint>
#include <cstring>

#include "ouster_b200.h"

namespace ouster {
namespace sdk {
namespace core {

#pragma pack(push, 1)
struct ZoneState {
    uint8_t live{0};
    uint8_t id{0};
    uint8_t error_flags{0};
    uint8_t trigger_type{0};
    uint8_t trigger_status{0};
    uint32_t triggered_frames{0};
    uint32_t count{0};
    uint32_t occlusion_count{0};
    uint32_t invalid_count{0};
    uint32_t max_count{0};
    uint32_t min_range{0};
    uint32_t max_range{0};
    uint32_t mean_range{0};
};
#pragma pack(pop)
static_assert(sizeof(ZoneState) == 37 && sizeof(ZoneState) == sizeof(ob_zone_state), "ZoneState is 37 bytes");

inline bool operator==(const ZoneState& a, const ZoneState& b) { return std::memcmp(&a, &b, sizeof(a)) == 0; }
inline bool operator!=(const ZoneState& a, const ZoneState& b) { return !(a == b); }

}  // namespace core
}  // namespace sdk
}  // namespace ouster
