// frame_ops.cpp -- the C++ frame operations (include/ouster/core/frame_ops.h) over the C ABI: field selection,
// the per-type visit rules and the reference's checks and texts here, the pixel work in ob_frame_mask_fields /
// ob_frame_select_rows on the GPU (ouster_core/src/frame_ops.cpp).
#include "ouster/core/frame_ops.h"

#include <cctype>
#include <cstring>
#include <regex>
#include <stdexcept>
#include <unordered_set>

#include "ouster/core/b200_runtime.h"

namespace ouster {
namespace sdk {
namespace core {

ProductInfo ProductInfo::create_product_info(const std::string& s) {
    ProductInfo pi;
    if (s.empty()) return pi;
    static const std::regex product_regex(
        R"(^(\w+)-(\d+|DOME)?(?:-(MAX))?(?:-(\d+))?(?:-(RGB))?(?:-((?!SR)\w+))?-?(SR)?)");
    std::smatch m;
    if (!std::regex_search(s, m, product_regex))
        throw std::runtime_error("Product Info \"" + s + "\" is not a recognized product info");
    pi.full_product_info = s;
    pi.form_factor = m.str(1) + m.str(2) + m.str(3);
    pi.short_range = !m.str(7).empty();
    pi.beam_config = m.str(6).empty() ? "U" : m.str(6);
    pi.rgb = m.str(5) == "RGB";
    try {
        pi.beam_count = std::stoi(m.str(4));
    } catch (const std::exception&) {
        pi.beam_count = 0;
    }
    return pi;
}

namespace frame_ops {
namespace {

bool handled(ChanFieldType t) {
    const int v = static_cast<int>(t);
    return v >= 1 && v <= 10;
}

std::string dims_message(size_t ndim) {
    return "Field: Eigen array conversion failed due to dimension mismatch. Underlying data has " +
           std::to_string(ndim) + " dimensions but must have 2 dimensions.";
}

// resolve_pixel_fields (frame_ops.cpp:19-62)
std::vector<std::string> resolve_pixel_fields(const LidarFrame& frame, const std::vector<std::string>* filtered) {
    std::unordered_set<std::string> pixel;
    for (const auto& ft : frame.field_types())
        if (ft.field_class == FieldClass::PIXEL_FIELD) pixel.insert(ft.name);
    std::vector<std::string> requested;
    if (filtered) {
        requested = *filtered;
    } else {
        for (const auto& kv : frame.fields()) requested.push_back(kv.first);
    }
    std::vector<std::string> present, non_pixel;
    for (const auto& f : requested) {
        if (!frame.has_field(f)) continue;
        if (!pixel.count(f)) {
            non_pixel.push_back(f);
            continue;
        }
        present.push_back(f);
    }
    if (filtered && !non_pixel.empty()) {
        std::string msg = "Only PIXEL_FIELD frame fields are supported here; requested non-pixel fields: [";
        for (size_t i = 0; i < non_pixel.size(); ++i) msg += (i ? ", " : "") + non_pixel[i];
        throw std::invalid_argument(msg + "]");
    }
    return present;
}

// the fields impl::visit_field_2d writes: handled types of shape (h, w); the dimension error for other handled ones
std::vector<ob_frame_field> targets(LidarFrame& frame, const std::vector<std::string>& names) {
    std::vector<ob_frame_field> out;
    for (const auto& n : names) {
        Field& f = frame.field(n);
        if (!handled(f.tag())) continue;
        if (f.shape().size() != 2) throw std::invalid_argument(dims_message(f.shape().size()));
        out.push_back(ob_frame_field{f.get(), static_cast<int32_t>(f.tag()), OB_FRAME_TARGET, 0, 0});
    }
    return out;
}

void run(LidarFrame& frame, ob_frame_predicate pred, std::vector<ob_frame_field>& fields, double lower,
         double upper, double invalid, const std::vector<int32_t>* shifts = nullptr) {
    if (fields.empty()) return;
    ob_frame_ops_io io{};
    io.n_frames = 1;
    io.h = static_cast<uint32_t>(frame.h);
    io.w = static_cast<uint32_t>(frame.w);
    io.predicate = pred;
    io.fields = fields.data();
    io.n_fields = fields.size();
    io.lower = lower;
    io.upper = upper;
    io.invalid = invalid;
    io.pixel_shift_by_row = shifts ? shifts->data() : nullptr;
    b200::check(ob_frame_mask_fields(&io, b200::thread_stream()));
    b200::synchronize();
}

void validate_beam_indices(const std::vector<size_t>& indices, size_t height) {
    if (indices.empty()) throw std::invalid_argument("beam indices can't be empty");
    std::unordered_set<size_t> seen;
    std::vector<size_t> bad;
    for (auto i : indices) {
        if (!seen.insert(i).second) throw std::invalid_argument("beam indices can't contain duplicates");
        if (i >= height) bad.push_back(i);
    }
    if (!bad.empty()) {
        std::string msg = "beam indices [";
        for (size_t i = 0; i < bad.size(); ++i) msg += (i ? ", " : "") + std::to_string(bad[i]);
        throw std::invalid_argument(msg + "] must be in the range [0, " + std::to_string(height) + ")");
    }
}

template <typename T>
std::vector<T> select_vector(const std::vector<T>& v, const std::vector<size_t>& idx) {
    std::vector<T> out;
    out.reserve(idx.size());
    for (auto i : idx) out.push_back(v.at(i));
    return out;
}

// form_factor_prod_line (frame_ops.cpp:110-124)
std::string form_factor_prod_line(const SensorInfo& metadata, size_t v_res) {
    const auto pi = ProductInfo::create_product_info(metadata.prod_line);
    auto ff = pi.form_factor;
    if (ff.find("MAX") != std::string::npos) {
        ff = "OS" + ff.substr(2, 1) + "MAX";
    } else if (!ff.empty() && std::isdigit(static_cast<unsigned char>(ff.back()))) {
        ff = ff.substr(0, ff.size() - 1) + "-" + ff.back();
    }
    ff += "-" + std::to_string(v_res);
    if (pi.rgb) ff += "-RGB";
    return ff;
}

}  // namespace

void clip(LidarFrame& frame, const std::vector<std::string>& fields, double lower, double upper, double invalid) {
    auto t = targets(frame, resolve_pixel_fields(frame, fields.empty() ? nullptr : &fields));
    run(frame, OB_FRAME_CLIP, t, lower, upper, invalid);
}

void filter_field(LidarFrame& frame, const std::string& field, double lower, double upper, double invalid,
                  const std::vector<std::string>* filtered_fields) {
    if (!frame.has_field(field)) throw std::out_of_range("Field '" + field + "' not found in LidarFrame.");
    Field& src = frame.field(field);
    if (src.shape().size() != 2 || src.shape()[0] != frame.h || src.shape()[1] != frame.w || !handled(src.tag()))
        throw std::invalid_argument("filter_field requires a pixel field with shape (h, w) to build a mask");
    auto t = targets(frame, resolve_pixel_fields(frame, filtered_fields));
    if (t.empty()) return;
    t.push_back(ob_frame_field{src.get(), static_cast<int32_t>(src.tag()), OB_FRAME_SOURCE, 0, 0});
    run(frame, OB_FRAME_VALUE, t, lower, upper, invalid);
}

void filter_uv(LidarFrame& frame, const std::string& coord_2d, size_t lower, size_t upper, double invalid,
               const std::vector<std::string>* filtered_fields) {
    if (coord_2d != "u" && coord_2d != "v")
        throw std::invalid_argument("coord_2d == " + coord_2d + " must be either 'u' or 'v'");
    const size_t size = coord_2d == "u" ? frame.h : frame.w;
    if (lower > size || upper > size)
        throw std::invalid_argument("lower == " + std::to_string(lower) + " and upper == " + std::to_string(upper) +
                                    " must be in the range [0, " + std::to_string(size) + "]");
    if (lower > upper)
        throw std::invalid_argument("lower == " + std::to_string(lower) + " must be less than upper == " +
                                    std::to_string(upper));
    const auto names = resolve_pixel_fields(frame, filtered_fields);
    auto t = targets(frame, names);
    if (coord_2d == "u") {
        run(frame, OB_FRAME_ROWS, t, double(lower), double(upper), invalid);
        return;
    }
    if (!frame.sensor_info) throw std::invalid_argument("filter_uv 'v' requires frame.sensor_info");
    // destagger() returns a zeroed field for a type the per-type visit skips, and the reference writes it back
    for (const auto& n : names) {
        Field& f = frame.field(n);
        if (handled(f.tag()) || f.bytes() == 0) continue;
        t.push_back(ob_frame_field{f.get(), static_cast<int32_t>(f.tag()), OB_FRAME_ZERO, 0,
                                   static_cast<uint32_t>(f.bytes() / (frame.h * frame.w))});
    }
    std::vector<int32_t> shifts(frame.sensor_info->format.pixel_shift_by_row.begin(),
                                frame.sensor_info->format.pixel_shift_by_row.end());
    if (shifts.size() != frame.h) throw std::invalid_argument("pixel_shift_by_row must have one entry per row");
    run(frame, OB_FRAME_COLS, t, double(lower), double(upper), invalid, &shifts);
}

void mask(LidarFrame& frame, const std::vector<std::string>& fields, ArrayRef<const uint8_t> mask) {
    if (mask.rows() != frame.h || mask.cols() != frame.w)
        throw std::invalid_argument("Used mask size doesn't match frame size");
    auto t = targets(frame, resolve_pixel_fields(frame, fields.empty() ? nullptr : &fields));
    if (t.empty()) return;
    t.push_back(ob_frame_field{const_cast<uint8_t*>(mask.data()), 1, OB_FRAME_SOURCE, 0, 0});
    run(frame, OB_FRAME_VALUE, t, 0.0, 0.0, 0.0);
}

std::vector<size_t> reduce_factor_to_indices(size_t factor, size_t height) {
    if (factor == 0) throw std::invalid_argument("factor == 0 can't be negative");
    if (height % factor != 0)
        throw std::invalid_argument("factor == " + std::to_string(factor) + " must be a divisor of " +
                                    std::to_string(height));
    if (factor == height) return {height / 2};
    std::vector<size_t> idx;
    for (size_t i = 0; i < height; i += factor) idx.push_back(i);
    return idx;
}

SensorInfo select_by_index_metadata(const SensorInfo& metadata, const std::vector<size_t>& indices) {
    validate_beam_indices(indices, metadata.h());
    SensorInfo out = metadata;
    out.prod_line = form_factor_prod_line(metadata, indices.size());
    out.format.pixels_per_column = static_cast<uint32_t>(indices.size());
    out.format.pixel_shift_by_row = select_vector(metadata.format.pixel_shift_by_row, indices);
    out.beam_azimuth_angles = select_vector(metadata.beam_azimuth_angles, indices);
    out.beam_altitude_angles = select_vector(metadata.beam_altitude_angles, indices);
    return out;
}

LidarFrame select_by_index(const LidarFrame& frame, const std::vector<size_t>& indices, bool update_metadata) {
    validate_beam_indices(indices, frame.h);
    if (!frame.sensor_info) throw std::invalid_argument("select_by_index requires frame.sensor_info");
    SensorInfo meta;
    if (update_metadata) meta = select_by_index_metadata(*frame.sensor_info, indices);
    LidarFrame result(indices.size(), frame.w, frame.field_types(), frame.sensor_info->format.columns_per_packet);
    result.frame_id = frame.frame_id;
    result.frame_status = frame.frame_status;
    result.shutdown_countdown = frame.shutdown_countdown;
    result.shot_limiting_countdown = frame.shot_limiting_countdown;
    auto copy_header = [](auto dst, auto src) {
        if (dst.size() == src.size() && src.size()) std::memcpy(dst.data(), src.data(), src.size() * sizeof(src[0]));
    };
    copy_header(result.timestamp(), frame.timestamp());
    copy_header(result.packet_timestamp(), frame.packet_timestamp());
    copy_header(result.measurement_id(), frame.measurement_id());
    copy_header(result.status(), frame.status());
    result.body_to_world() = frame.body_to_world();
    std::vector<ob_frame_rows_entry> rows;
    for (const auto& ft : frame.field_types()) {
        const Field& src = frame.field(ft.name);
        if (ft.field_class != FieldClass::PIXEL_FIELD) {
            result.field(ft.name) = src;
            continue;
        }
        if (src.shape().empty()) throw std::invalid_argument("cannot select rows from non-array fields");
        Field& dst = result.field(ft.name);
        if (dst.shape()[0] != indices.size()) throw std::invalid_argument("selected field height mismatch");
        rows.push_back(ob_frame_rows_entry{src.get(), dst.get(), frame.h ? src.bytes() / frame.h : 0, frame.h});
    }
    std::vector<uint32_t> idx(indices.begin(), indices.end());
    ob_frame_rows_io io{rows.data(), static_cast<uint32_t>(rows.size()), static_cast<uint32_t>(idx.size()),
                        idx.data()};
    b200::check(ob_frame_select_rows(&io, b200::thread_stream()));
    b200::synchronize();
    if (update_metadata) result.sensor_info = std::make_shared<SensorInfo>(meta);
    return result;
}

SensorInfo reduce_by_factor_metadata(const SensorInfo& metadata, size_t factor) {
    return select_by_index_metadata(metadata, reduce_factor_to_indices(factor, metadata.h()));
}

LidarFrame reduce_by_factor(const LidarFrame& frame, size_t factor, bool update_metadata) {
    return select_by_index(frame, reduce_factor_to_indices(factor, frame.h), update_metadata);
}

}  // namespace frame_ops
}  // namespace core
}  // namespace sdk
}  // namespace ouster
