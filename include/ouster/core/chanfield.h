// chanfield.h -- channel field names and element type tags
// (mirrors ouster_core/include/ouster/core/chanfield.h:20-170).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

#include "ouster/core/visibility.h"

namespace ouster {
namespace sdk {
namespace core {

namespace ChanField {
static constexpr const char* RANGE = "RANGE";
static constexpr const char* RANGE2 = "RANGE2";
static constexpr const char* SIGNAL = "SIGNAL";
static constexpr const char* SIGNAL2 = "SIGNAL2";
static constexpr const char* REFLECTIVITY = "REFLECTIVITY";
static constexpr const char* REFLECTIVITY2 = "REFLECTIVITY2";
static constexpr const char* NEAR_IR = "NEAR_IR";
static constexpr const char* FLAGS = "FLAGS";
static constexpr const char* FLAGS2 = "FLAGS2";
static constexpr const char* WINDOW = "WINDOW";
static constexpr const char* ZONE_MASK = "ZONE_MASK";
static constexpr const char* R = "R";
static constexpr const char* G = "G";
static constexpr const char* B = "B";
static constexpr const char* RGB = "RGB";
static constexpr const char* RAW_HEADERS = "RAW_HEADERS";
static constexpr const char* RAW32_WORD1 = "RAW32_WORD1";
static constexpr const char* RAW32_WORD2 = "RAW32_WORD2";
static constexpr const char* RAW32_WORD3 = "RAW32_WORD3";
static constexpr const char* RAW32_WORD4 = "RAW32_WORD4";
static constexpr const char* RAW32_WORD5 = "RAW32_WORD5";
static constexpr const char* NORMALS = "NORMALS";
static constexpr const char* NORMALS2 = "NORMALS2";
static constexpr const char* GROUND = "GROUND";
static constexpr const char* GROUND2 = "GROUND2";
/// The field of return `ret` (0-based): `base` for the first return, then base + "2", base + "3", ...
inline std::string return_field_name(const std::string& base, int ret) {
    return ret <= 0 ? base : base + std::to_string(ret + 1);
}
}  // namespace ChanField

enum class ChanFieldType {
    VOID = 0,
    UINT8 = 1,
    UINT16 = 2,
    UINT32 = 3,
    UINT64 = 4,
    INT8 = 5,
    INT16 = 6,
    INT32 = 7,
    INT64 = 8,
    FLOAT32 = 9,
    FLOAT64 = 10,
    CHAR = 11,
    FLOAT16 = 12,
    ZONE_STATE = 30,
    UNREGISTERED = 100
};

/// Size in bytes of one element of the given type (0 for VOID/unknown).
OUSTER_API_FUNCTION size_t field_type_size(ChanFieldType ft);
/// All-ones mask of the type's width.
OUSTER_API_FUNCTION uint64_t field_type_mask(ChanFieldType ft);
OUSTER_API_FUNCTION std::string to_string(ChanFieldType ft);

/// 16-bit float storage type (bit pattern only; the path never does arithmetic on it).
struct float16_t {
    uint16_t bits{0};
    float16_t() = default;
    explicit float16_t(uint16_t b) : bits(b) {}
    bool operator==(const float16_t& o) const { return bits == o.bits; }
};
namespace impl {
/// three packed float16 (RGB pixel), reference: impl::float3x16_t
struct float3x16_t {
    uint16_t v[3];
};
}  // namespace impl

template <typename T>
struct FieldTag;
template <> struct FieldTag<uint8_t> { static constexpr ChanFieldType tag = ChanFieldType::UINT8; };
template <> struct FieldTag<uint16_t> { static constexpr ChanFieldType tag = ChanFieldType::UINT16; };
template <> struct FieldTag<uint32_t> { static constexpr ChanFieldType tag = ChanFieldType::UINT32; };
template <> struct FieldTag<uint64_t> { static constexpr ChanFieldType tag = ChanFieldType::UINT64; };
template <> struct FieldTag<int8_t> { static constexpr ChanFieldType tag = ChanFieldType::INT8; };
template <> struct FieldTag<int16_t> { static constexpr ChanFieldType tag = ChanFieldType::INT16; };
template <> struct FieldTag<int32_t> { static constexpr ChanFieldType tag = ChanFieldType::INT32; };
template <> struct FieldTag<int64_t> { static constexpr ChanFieldType tag = ChanFieldType::INT64; };
template <> struct FieldTag<float> { static constexpr ChanFieldType tag = ChanFieldType::FLOAT32; };
template <> struct FieldTag<double> { static constexpr ChanFieldType tag = ChanFieldType::FLOAT64; };
template <> struct FieldTag<float16_t> { static constexpr ChanFieldType tag = ChanFieldType::FLOAT16; };

}  // namespace core
}  // namespace sdk
}  // namespace ouster
