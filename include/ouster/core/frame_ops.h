// frame_ops.h -- drop-in for ouster_core/include/ouster/core/frame_ops.h (DESIGN f-10): the nine functions of
// namespace frame_ops with the reference's signatures, defaults and exception texts, on the host LidarFrame.
// The pixel work runs on the GPU through ob_frame_mask_fields / ob_frame_select_rows: the fields are staged to the
// device, written there and copied back before the call returns.
//
// Differences from the reference (DESIGN §9): `mask` takes an ArrayRef<const uint8_t> (h x w) where the reference
// takes Eigen::Ref<const img_t<uint8_t>>; every argument is checked before anything is written, so a call that
// throws leaves the frame as it was; an `invalid` the reference's static_cast<T> leaves undefined (NaN or infinite
// for an integer field, or out of the type's range after truncation) throws std::invalid_argument.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "ouster/core/lidar_frame.h"
#include "ouster/core/sensor_info.h"
#include "ouster/core/typedefs.h"
#include "ouster/core/visibility.h"

namespace ouster {
namespace sdk {
namespace core {

/// ProductInfo::create_product_info (sensor_info.cpp:442-470): the parts of a product line string.
struct OUSTER_API_CLASS ProductInfo {
    std::string full_product_info;
    std::string form_factor;
    bool short_range{false};
    std::string beam_config;
    int beam_count{0};
    bool rgb{false};
    /// throws std::runtime_error("Product Info \"X\" is not a recognized product info")
    OUSTER_API_FUNCTION static ProductInfo create_product_info(const std::string& product_info_string);
};

namespace frame_ops {

/// Values of the pixel fields (all of them when `fields` is empty) outside [lower, upper] become invalid.
OUSTER_API_FUNCTION void clip(LidarFrame& frame, const std::vector<std::string>& fields, double lower, double upper,
                              double invalid = 0);

/// Pixels whose `field` value lies inside [lower, upper] become invalid in the filtered fields (all pixel fields
/// when null).
OUSTER_API_FUNCTION void filter_field(LidarFrame& frame, const std::string& field, double lower, double upper,
                                      double invalid = 0,
                                      const std::vector<std::string>* filtered_fields = nullptr);

/// Rows ("u") or destaggered columns ("v") in [lower, upper) become invalid.
OUSTER_API_FUNCTION void filter_uv(LidarFrame& frame, const std::string& coord_2d, size_t lower, size_t upper,
                                   double invalid = 0, const std::vector<std::string>* filtered_fields = nullptr);

/// Pixels whose mask byte is 0 become 0 in the fields (all pixel fields when empty).
OUSTER_API_FUNCTION void mask(LidarFrame& frame, const std::vector<std::string>& fields,
                              ArrayRef<const uint8_t> mask);

OUSTER_API_FUNCTION std::vector<size_t> reduce_factor_to_indices(size_t factor, size_t height);

OUSTER_API_FUNCTION SensorInfo select_by_index_metadata(const SensorInfo& metadata,
                                                        const std::vector<size_t>& indices);

/// The selected rows of every pixel field; headers and other fields copied.  sensor_info is null unless
/// update_metadata, as in the reference.
OUSTER_API_FUNCTION LidarFrame select_by_index(const LidarFrame& frame, const std::vector<size_t>& indices,
                                               bool update_metadata = false);

OUSTER_API_FUNCTION SensorInfo reduce_by_factor_metadata(const SensorInfo& metadata, size_t factor);

OUSTER_API_FUNCTION LidarFrame reduce_by_factor(const LidarFrame& frame, size_t factor,
                                                bool update_metadata = false);

}  // namespace frame_ops
}  // namespace core
}  // namespace sdk
}  // namespace ouster
