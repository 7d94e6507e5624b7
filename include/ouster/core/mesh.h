// mesh.h -- core::Mesh (mirrors ouster_core/include/ouster/core/mesh.h and src/mesh.cpp:41-294; DESIGN f-8): the
// triangles of a zone's STL, loaded on the host with the reference's acceptance rules, and its bounding sphere.
//
// Loading: a file is ASCII when "endsolid" (any case) starts after the 80-byte header, else binary.
//  * ASCII: lines are trimmed of ' ', '\t', '\r', blank and '#' lines skipped, and lower-cased.  "solid" opens the
//    file; then "facet ..." blocks of "outer loop", three "vertex x y z" lines, "endloop", "endfacet", until
//    "endsolid".  Anything else, or the end of the file first, is an error.  Numbers go through std::stof, so a
//    number it cannot convert throws as in the reference.
//  * binary: an 80-byte header, a uint32 triangle count and 50-byte records (normal, three vertices, a 2-byte
//    attribute count, which the last record may lack).
// Errors print "STL Parsing Error: ..." on stderr and make the load return false.
//
// Zone::render (zone.h) runs the ray tests on the GPU; intersects_with_bounding_sphere(),
// closest_and_farthest_intersections() and intersection_distances() are the host forms, for single rays.
#pragma once
#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>
#include <set>
#include <sstream>
#include <string>
#include <utility>
#include <vector>

#include "ouster/core/coord.h"
#include "ouster/core/triangle.h"

namespace ouster {
namespace sdk {
namespace core {

namespace zone_detail {

inline void stl_error(const std::string& message, const std::string& line = "") {
    std::cerr << "STL Parsing Error: " << message;
    if (!line.empty()) std::cerr << ": '" << line << "'";
    std::cerr << std::endl;
}

inline bool is_word_char(char c) { return std::isalnum(static_cast<unsigned char>(c)) || c == '_'; }
inline bool is_space(char c) { return std::isspace(static_cast<unsigned char>(c)) != 0; }

// `line` (already trimmed) starts with `word`; with `whole`, not followed by a word character
inline bool starts_with(const std::string& line, const char* word, bool whole) {
    const size_t n = std::strlen(word);
    if (line.compare(0, n, word) != 0) return false;
    return !whole || line.size() == n || !is_word_char(line[n]);
}

// "outer", one or more spaces, "loop"
inline bool is_outer_loop(const std::string& line) {
    if (!starts_with(line, "outer", false)) return false;
    size_t i = 5;
    if (i >= line.size() || !is_space(line[i])) return false;
    while (i < line.size() && is_space(line[i])) ++i;
    return line.compare(i, 4, "loop") == 0;
}

// a number token: optional '-', one or more of [0-9.], then an exponent only if [eE][+-]digits follows
inline bool number_token(const std::string& s, size_t& i, std::string& out) {
    const size_t start = i;
    if (i < s.size() && s[i] == '-') ++i;
    const size_t body = i;
    while (i < s.size() && (std::isdigit(static_cast<unsigned char>(s[i])) || s[i] == '.')) ++i;
    if (i == body) {
        i = start;
        return false;
    }
    if (i + 2 < s.size() && (s[i] == 'e' || s[i] == 'E') && (s[i + 1] == '+' || s[i + 1] == '-') &&
        std::isdigit(static_cast<unsigned char>(s[i + 2]))) {
        i += 2;
        while (i < s.size() && std::isdigit(static_cast<unsigned char>(s[i]))) ++i;
    }
    out = s.substr(start, i - start);
    return true;
}

// "vertex" and three numbers separated by whitespace; whatever follows the third is ignored
inline bool parse_vertex(const std::string& line, Coord& out) {
    if (!starts_with(line, "vertex", false)) return false;
    size_t i = 6;
    for (int k = 0; k < 3; ++k) {
        if (i >= line.size() || !is_space(line[i])) return false;
        while (i < line.size() && is_space(line[i])) ++i;
        std::string tok;
        if (!number_token(line, i, tok)) return false;
        out[k] = std::stof(tok);
    }
    return true;
}

class AsciiLines {
   public:
    explicit AsciiLines(const std::string& text) : in_(text) {}
    bool next(std::string& line) {
        while (std::getline(in_, line)) {
            const size_t b = line.find_first_not_of(" \t\r");
            if (b == std::string::npos) continue;
            const size_t e = line.find_last_not_of(" \t\r");
            line = line.substr(b, e - b + 1);
            if (line[0] == '#') continue;
            for (char& c : line) c = static_cast<char>(std::tolower(static_cast<unsigned char>(c)));
            return true;
        }
        line.clear();
        return false;
    }

   private:
    std::istringstream in_;
};

}  // namespace zone_detail

class Mesh {
   public:
    Mesh() = default;
    explicit Mesh(const std::vector<Triangle>& tris) : triangles_(tris) { update_sphere(); }
    explicit Mesh(std::vector<Triangle>&& tris) : triangles_(std::move(tris)) { update_sphere(); }

    bool load_from_stl(const std::string& path) {
        std::ifstream in(path, std::ios::in | std::ios::binary);
        return load_from_stl_stream(in);
    }
    bool load_from_stl_bytes(const std::vector<uint8_t>& bytes) {
        return load(std::string(bytes.begin(), bytes.end()));
    }
    bool load_from_stl_stream(std::istream& in) {
        std::string data((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
        return load(data);
    }

    const std::vector<Triangle>& triangles() const { return triangles_; }
    /// (centroid, radius): the centroid is the sequential float sum of every vertex divided by 3n, the radius the
    /// square root of the largest squared distance of a vertex from it.
    const std::pair<Coord, float>& bounding_sphere() const { return sphere_; }

    bool intersects_with_bounding_sphere(const Ray& beam) const {
        const Coord oc = beam.offset - sphere_.first;
        const float b = oc.dot(beam.direction);
        const float c = oc.dot(oc) - sphere_.second * sphere_.second;
        if (c > 0.0f && b > 0.0f) return false;
        volatile float disc = b * b - c;  // as written: a NaN discriminant is a miss
        return disc >= 0.0f;
    }
    std::multiset<float> intersection_distances(const Ray& beam) const {
        std::multiset<float> d;
        for (const auto& t : triangles_) {
            const float x = t.intersect(beam);
            if (x > 0) d.insert(x);
        }
        return d;
    }
    /// (nearest, farthest) hit; (0, t) for a single hit; false without a hit
    bool closest_and_farthest_intersections(const Ray& beam, BoundsF& z) const {
        if (!intersects_with_bounding_sphere(beam)) return false;
        const auto d = intersection_distances(beam);
        if (d.empty()) return false;
        z.first = d.size() > 1 ? *d.begin() : 0.0f;
        z.second = *d.rbegin();
        return true;
    }

    bool operator==(const Mesh& o) const { return triangles_ == o.triangles_; }
    bool operator!=(const Mesh& o) const { return !(*this == o); }

   private:
    static constexpr size_t kHeader = 80;

    bool load(const std::string& data) {
        std::string lower(data);
        for (char& c : lower) c = static_cast<char>(std::tolower(static_cast<unsigned char>(c)));
        const size_t pos = lower.find("endsolid");
        const bool ascii = pos != std::string::npos && pos > kHeader;
        std::vector<Triangle> tris;
        if (!(ascii ? load_ascii(data, tris) : load_binary(data, tris))) return false;
        triangles_ = std::move(tris);
        update_sphere();
        return true;
    }

    static bool load_ascii(const std::string& data, std::vector<Triangle>& tris) {
        using namespace zone_detail;
        AsciiLines lines(data);
        std::string line;
        if (!lines.next(line) || !starts_with(line, "solid", true)) {
            stl_error("Failed to find 'solid' header", line);
            return false;
        }
        while (lines.next(line)) {
            if (starts_with(line, "facet", true)) {
                Coord v[3];
                if (!lines.next(line) || !is_outer_loop(line)) {
                    stl_error("Expected 'outer loop'", line);
                    return false;
                }
                for (int k = 0; k < 3; ++k) {
                    if (!lines.next(line) || !parse_vertex(line, v[k])) {
                        stl_error("Expected 'vertex'", line);
                        return false;
                    }
                }
                if (!lines.next(line) || !starts_with(line, "endloop", false)) {
                    stl_error("Expected 'endloop'", line);
                    return false;
                }
                if (!lines.next(line) || !starts_with(line, "endfacet", false)) {
                    stl_error("Expected 'endfacet'", line);
                    return false;
                }
                tris.emplace_back(v[0], v[1], v[2]);
            } else if (starts_with(line, "endsolid", true)) {
                return true;
            } else {
                stl_error("Unexpected line outside of a facet", line);
                return false;
            }
        }
        stl_error("File ended unexpectedly without 'endsolid'");
        return false;
    }

    static bool load_binary(const std::string& data, std::vector<Triangle>& tris) {
        if (data.size() < kHeader) {
            zone_detail::stl_error("File too short.");
            return false;
        }
        if (data.size() < kHeader + 4) {
            zone_detail::stl_error("Unknown # of n_tris.");
            return false;
        }
        uint32_t n = 0;
        std::memcpy(&n, data.data() + kHeader, 4);
        for (uint32_t i = 0; i < n; ++i) {
            const size_t at = kHeader + 4 + size_t(50) * i;
            if (data.size() < at + 48) {
                zone_detail::stl_error("Mismatch in # of n_tris.");
                return false;
            }
            float f[12];
            std::memcpy(f, data.data() + at, sizeof(f));
            tris.emplace_back(Coord(f + 3), Coord(f + 6), Coord(f + 9));
        }
        return true;
    }

    void update_sphere() {
        Coord c{0, 0, 0};
        for (const auto& t : triangles_)
            for (int k = 0; k < 3; ++k) c += t.coords[k];
        c = c / static_cast<float>(3 * triangles_.size());
        float r2 = 0;
        for (const auto& t : triangles_) {
            float m = (t.coords[0] - c).squaredNorm();  // the first of the largest, by operator<
            const float b = (t.coords[1] - c).squaredNorm(), d = (t.coords[2] - c).squaredNorm();
            if (m < b) m = b;
            if (m < d) m = d;
            if (m < r2) m = r2;
            r2 = m;
        }
        sphere_ = {c, std::sqrt(r2)};
    }

    std::vector<Triangle> triangles_;
    std::pair<Coord, float> sphere_{};
};

}  // namespace core
}  // namespace sdk
}  // namespace ouster
