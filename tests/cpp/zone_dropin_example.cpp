// zone_dropin_example.cpp -- user code written against ouster_core's Mesh, Zone, BeamConfig, Zrb and ZoneState the
// way the reference's tests use them, compiled against the replacement headers and run on the GPU.
//   zone_dropin_example <stl_dir> <beams.txt> <out.bin>
// beams.txt: "h w", h altitudes, h azimuths (degrees), beam_to_lidar and lidar_to_sensor (16 row-major each).
// Loads the STL fixtures, checks the parser's verdicts and the error texts, renders 0.stl in the BODY frame
// (sensor_to_body z = 1 m) and writes near then far (h x w uint32 each) to out.bin.  Prints "ZONE DROPIN OK".
// Built and run by tests/test_gpu_zone_dropin.py.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "ouster/core/zone.h"
#include "ouster/core/zone_state.h"

using namespace ouster::sdk::core;

#define CHECK(cond)                                                                      \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            std::exit(1);                                                                \
        }                                                                                \
    } while (0)

template <typename F>
static void expect_logic_error(F&& fn, const std::string& text) {
    try {
        fn();
    } catch (const std::logic_error& e) {
        if (std::string(e.what()) != text) {
            std::fprintf(stderr, "wrong message: '%s' (wanted '%s')\n", e.what(), text.c_str());
            std::exit(1);
        }
        return;
    }
    std::fprintf(stderr, "expected std::logic_error '%s'\n", text.c_str());
    std::exit(1);
}

int main(int argc, char** argv) {
    CHECK(argc == 4);
    const std::string dir = argv[1];
    // mesh_test.cpp: binary, ASCII and SolidWorks files load; the malformed ones do not
    Mesh mesh;
    CHECK(mesh.load_from_stl(dir + "/0.stl") && mesh.triangles().size() == 12);
    Mesh ascii;
    CHECK(ascii.load_from_stl(dir + "/ascii.stl") && ascii.triangles().size() == 12);
    CHECK(ascii.triangles()[0].coords[0] == Coord(-20, -20, 40));
    CHECK(ascii.triangles()[0].normal == Coord(0, 0, 1));
    Mesh sw;
    CHECK(sw.load_from_stl(dir + "/solidworks_binary.stl") && sw.triangles().size() == 12);
    Mesh empty;
    CHECK(empty.load_from_stl(dir + "/empty.stl") && empty.triangles().empty());
    for (const char* bad : {"ascii_invalid_expected_vertex.stl", "ascii_invalid_expected_endloop.stl",
                            "ascii_invalid_expected_outer_loop.stl", "ascii_invalid_expected_endfacet.stl",
                            "ascii_empty.stl", "ascii_invalid_expected_solid.stl",
                            "ascii_invalid_expected_endsolid.stl", "ascii_invalid_unexpected_line.stl"}) {
        Mesh m;
        CHECK(!m.load_from_stl(dir + "/" + bad));
    }
    // mesh_test.cpp bounding_sphere
    Mesh three({Triangle({1, 1, 1}, {1, 1, 1}, {1, 1, 1}), Triangle({2, 2, 2}, {2, 2, 2}, {2, 2, 2}),
                Triangle({2, 2, 2}, {2, 2, 2}, {2, 2, 2})});
    CHECK(std::fabs(three.bounding_sphere().second - 1.1547004f) < 1e-6f);
    CHECK(three.intersects_with_bounding_sphere(Ray{{0, 0, 0}, Coord(1, 1, 1).normalized()}));
    CHECK(!three.intersects_with_bounding_sphere(Ray{{0, 0, 0}, Coord(-1, -1, -1).normalized()}));

    // the beams
    std::ifstream in(argv[2]);
    uint32_t h = 0, w = 0;
    in >> h >> w;
    std::vector<double> alt(h), az(h);
    for (auto& v : alt) in >> v;
    for (auto& v : az) in >> v;
    mat4d b2l, l2s;
    for (auto& v : b2l.m) in >> v;
    for (auto& v : l2s.m) in >> v;
    CHECK(in.good());
    mat4d s2b = mat4d::Identity();
    s2b(2, 3) = 1.0;
    BeamConfig config(w, alt, az, b2l, l2s, s2b, DEFAULT_M_PER_ZMBIN, 122222000785ull);
    BeamConfig no_body(w, alt, az, b2l, l2s, std::nullopt);

    Zone zone;
    zone.stl = Stl(dir + "/0.stl");
    zone.stl->coordinate_frame = Stl::CoordinateFrame::BODY;
    expect_logic_error([&] { zone.render(config); }, "Zone: point_count must be in [1, 262143]");
    zone.point_count = 1;
    zone.frame_count = 1;
    expect_logic_error([&] { zone.render(config); }, "Zone: mode must be OCCUPANCY or VACANCY");
    zone.mode = Zone::ZoneMode::OCCUPANCY;
    CHECK(!zone.render(no_body));  // BODY frame without a sensor_to_body_transform
    CHECK(zone.render(config));
    CHECK(zone.zrb && zone.zrb->near_range_mm.rows() == h && zone.zrb->near_range_mm.cols() == w);
    CHECK(zone.zrb->serial_number == 122222000785ull && zone.zrb->sensor_to_body_transform == s2b);
    size_t hit = 0;
    for (size_t i = 0; i < zone.zrb->far_range_mm.size(); ++i) hit += zone.zrb->far_range_mm(i) != 0;
    CHECK(hit > 0);
    Zone big = zone;
    big.zrb.reset();  // check_invariants would test the old ZRB's area first
    big.point_count = static_cast<uint32_t>(h * w);
    expect_logic_error([&] { big.render(config); }, "Zone: area of rendered zone (" + std::to_string(hit) +
                                                        ") is smaller than point_count (" +
                                                        std::to_string(h * w) + ") specified in zone.");
    std::ofstream out(argv[3], std::ios::binary);
    out.write(reinterpret_cast<const char*>(zone.zrb->near_range_mm.data()), h * w * 4);
    out.write(reinterpret_cast<const char*>(zone.zrb->far_range_mm.data()), h * w * 4);
    CHECK(out.good());

    ZoneState a{}, b{};
    b.id = 255;
    CHECK(sizeof(ZoneState) == 37 && a != b && to_string(Zone::ZoneMode::VACANCY) == "VACANCY");
    std::printf("ZONE DROPIN OK (%zu pixels hit)\n", hit);
    return 0;
}
