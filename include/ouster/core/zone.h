// zone.h -- core::Zone, Stl and ZoneMode (mirrors ouster_core/include/ouster/core/zone.h, stl.h and
// src/zone.cpp:18-135; DESIGN f-8).  Zone::render casts every beam of a BeamConfig against the zone's STL mesh on
// the GPU (ob_zone_render) and stores the nearest and farthest hits as the Zrb's near / far range images in mm.
// Stl keeps the file's bytes and the zone's coordinate frame; its hash, and ZRB / ZoneSet files, are not provided.
#pragma once
#include <cstdint>
#include <fstream>
#include <iostream>
#include <iterator>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/beam_config.h"
#include "ouster/core/mesh.h"
#include "ouster/core/zrb.h"

namespace ouster {
namespace sdk {
namespace core {

class Stl {
   public:
    enum class CoordinateFrame : uint8_t { NONE = 0, BODY = 1, SENSOR = 2 };

    Stl() = default;
    explicit Stl(const std::string& path) {
        std::ifstream in(path, std::ios::in | std::ios::binary);
        if (!in) throw std::runtime_error("Stl: failed to open " + path);
        blob_.assign(std::istreambuf_iterator<char>(in), std::istreambuf_iterator<char>());
    }
    explicit Stl(const std::vector<uint8_t>& blob) : blob_(blob) {}

    const std::vector<uint8_t>& blob() const { return blob_; }
    /// the mesh of the blob; throws std::runtime_error when it does not parse
    Mesh to_mesh() const {
        Mesh m;
        if (!m.load_from_stl_bytes(blob_)) throw std::runtime_error("Stl: failed to parse STL");
        return m;
    }
    bool operator==(const Stl& o) const { return blob_ == o.blob_ && coordinate_frame == o.coordinate_frame; }

    CoordinateFrame coordinate_frame{CoordinateFrame::NONE};

   private:
    std::vector<uint8_t> blob_;
};

class Zone {
   public:
    static constexpr uint32_t MAX_TRIANGLES = OB_ZONE_MAX_TRIANGLES;
    enum class ZoneMode : uint8_t { NONE = 0, OCCUPANCY = 1, VACANCY = 2 };

    uint32_t point_count{};
    uint32_t frame_count{};
    ZoneMode mode{ZoneMode::NONE};
    std::optional<Stl> stl;
    std::optional<Zrb> zrb;

    static bool string_to_zonemode(const std::string& str, ZoneMode& out) {
        if (str == "OCCUPANCY") {
            out = ZoneMode::OCCUPANCY;
        } else if (str == "VACANCY") {
            out = ZoneMode::VACANCY;
        } else {
            return false;
        }
        return true;
    }

    /// @throws std::logic_error with the reference's texts
    void check_invariants() const {
        if (point_count == 0) throw std::logic_error("Zone: point_count must be in [1, 262143]");
        if (frame_count == 0) throw std::logic_error("Zone: frame_count must be in [1, 65535]");
        if (!stl && !zrb) throw std::logic_error("Zone: must have either STL or ZRB");
        if (mode != ZoneMode::OCCUPANCY && mode != ZoneMode::VACANCY)
            throw std::logic_error("Zone: mode must be OCCUPANCY or VACANCY");
        if (stl) {
            if (stl->blob().empty()) throw std::logic_error("Zone: STL blob cannot be empty");
            if (stl->coordinate_frame == Stl::CoordinateFrame::NONE)
                throw std::logic_error("Zone: STL coordinate frame must be BODY or SENSOR");
        }
        if (zrb) {
            size_t nonzero = 0;
            for (size_t i = 0; i < zrb->far_range_mm.size(); ++i) nonzero += zrb->far_range_mm(i) != 0;
            if (nonzero < point_count)
                throw std::logic_error("Zone: ZRB far range image has fewer nonzero pixels than point_count");
        }
    }

    /// Render the STL against the config's beams on the GPU into a new zrb.  Returns false, after a message on
    /// stderr, without an STL, with 0 or more than MAX_TRIANGLES triangles, for a BODY zone without a
    /// sensor_to_body_transform, or when no beam meets the zone.
    /// @throws std::logic_error from check_invariants(), "Zone::render: range overflow" and
    ///         "Zone: area of rendered zone (N) is smaller than point_count (M) specified in zone."
    bool render(const BeamConfig& config) {
        check_invariants();
        if (!stl) {
            std::cerr << "Zone: Error rendering zone, no STL provided.\n";
            return false;
        }
        const Mesh mesh = stl->to_mesh();
        const auto& tris = mesh.triangles();
        if (tris.empty()) {
            std::cerr << "Zone: Error rendering zone, STL has no triangles.\n";
            return false;
        }
        if (tris.size() > MAX_TRIANGLES) {
            std::cerr << "Zone: Error rendering zone, STL has too many triangles.\n";
            return false;
        }
        const bool body = stl->coordinate_frame == Stl::CoordinateFrame::BODY;
        if (body && !config.sensor_to_body_transform) {
            std::cerr << "Zone: Error rendering zone, sensor_to_body_transform not set for BODY coordinate frame.\n";
            return false;
        }
        std::vector<float> packed(tris.size() * 9);
        for (size_t t = 0; t < tris.size(); ++t)
            for (int v = 0; v < 3; ++v)
                for (int k = 0; k < 3; ++k) packed[9 * t + 3 * v + k] = tris[t].coords[v][k];
        ob_zone_desc desc{};
        desc.triangles = packed.data();
        desc.n_triangles = static_cast<uint32_t>(tris.size());
        desc.coordinate_frame = static_cast<int32_t>(stl->coordinate_frame);
        desc.point_count = point_count;
        desc.frame_count = frame_count;
        desc.mode = static_cast<int32_t>(mode);
        Zrb out(config.n_rows, config.n_cols, config.m_per_zmbin, config.serial_number,
                config.beam_to_lidar_transform, config.lidar_to_sensor_transform,
                config.sensor_to_body_transform.value_or(mat4d::Identity()));
        ob_zone_render_io io{};
        io.n_rows = config.n_rows;
        io.n_cols = config.n_cols;
        void *dir = nullptr, *off = nullptr;
        b200::check(ob_lut_device_ptrs(config.lut_no_sensor_to_body_transform.get(), &dir, &off));
        io.sensor_direction = static_cast<const double*>(dir);
        io.sensor_offset = static_cast<const double*>(off);
        if (config.lut) {
            b200::check(ob_lut_device_ptrs(config.lut.get(), &dir, &off));
            io.body_direction = static_cast<const double*>(dir);
            io.body_offset = static_cast<const double*>(off);
        }
        io.zones = &desc;
        io.n_zones = 1;
        io.near_mm = out.near_range_mm.data();
        io.far_mm = out.far_range_mm.data();
        uint32_t hits = 0;
        io.pixels_with_intersections = &hits;
        const ob_status st = ob_zone_render(&io, b200::thread_stream());
        if (st == OB_RUNTIME_ERROR) throw std::logic_error(ob_last_error());  // overflow / area, as the reference
        b200::check(st);
        zrb = std::move(out);
        return hits > 0;
    }
};

inline std::string to_string(Zone::ZoneMode zone_mode) {
    switch (zone_mode) {
        case Zone::ZoneMode::NONE: return "NONE";
        case Zone::ZoneMode::OCCUPANCY: return "OCCUPANCY";
        case Zone::ZoneMode::VACANCY: return "VACANCY";
    }
    return "UNKNOWN";
}

}  // namespace core
}  // namespace sdk
}  // namespace ouster
