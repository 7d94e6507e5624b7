/*
 * orc_zone.c -- CPU oracle of zone monitoring: Zone::render and the per-frame occupancy of EmulatedZoneMon.
 * TEST INFRASTRUCTURE ONLY.  A plain-C restatement of the reference's arithmetic, compiled with
 * -ffp-contract=off so every float operation rounds on its own as it does in the reference's x86 build.
 * Paths are relative to the reference tree.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef struct {
    float x, y, z;
} v3;

static v3 sub(v3 a, v3 b) {
    v3 r = {a.x - b.x, a.y - b.y, a.z - b.z};
    return r;
}
/* Eigen's cross (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0) */
static v3 cross(v3 a, v3 b) {
    v3 r = {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
    return r;
}
/* Eigen's dot of 3: (x0 y0 + x1 y1) + x2 y2 */
static float dot(v3 a, v3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
static v3 at(const float* p) {
    v3 r = {p[0], p[1], p[2]};
    return r;
}

/* Triangle::intersect, ouster_core/src/triangle.cpp:19-50.  tri: v0, v1, v2 (9 floats). */
float orc_tri_intersect(const float* tri, const float* offset, const float* direction) {
    const float epsilon = FLT_EPSILON;
    const v3 o = at(offset), d = at(direction), c0 = at(tri), c1 = at(tri + 3), c2 = at(tri + 6);
    const v3 edge1 = sub(c1, c0), edge2 = sub(c2, c0);
    const v3 ray_cross_e2 = cross(d, edge2);
    const float det = dot(edge1, ray_cross_e2);
    if (det > -epsilon && det < epsilon) return -FLT_MAX;
    const float inv_det = 1.0f / det;
    const v3 s = sub(o, c0);
    const float u = inv_det * dot(s, ray_cross_e2);
    if ((u < 0 && fabsf(u) > epsilon) || (u > 1 && fabsf(u - 1) > epsilon)) return -FLT_MAX;
    const v3 s_cross_e1 = cross(s, edge1);
    const float v = inv_det * dot(d, s_cross_e1);
    if ((v < 0 && fabsf(v) > epsilon) || (u + v > 1 && fabsf(u + v - 1) > epsilon)) return -FLT_MAX;
    return inv_det * dot(edge2, s_cross_e1);
}

/* compute_centroid / compute_bounding_sphere, mesh.cpp:41-60.  out: cx, cy, cz, radius */
void orc_bounding_sphere(const float* tris, size_t n, float* out) {
    v3 c = {0, 0, 0};
    for (size_t i = 0; i < n; ++i)
        for (int k = 0; k < 3; ++k) {
            c.x += tris[9 * i + 3 * k];
            c.y += tris[9 * i + 3 * k + 1];
            c.z += tris[9 * i + 3 * k + 2];
        }
    const float denom = (float)(3 * n); /* Coord / size_t: the scalar converts to float */
    c.x = c.x / denom;
    c.y = c.y / denom;
    c.z = c.z / denom;
    float r2 = 0;
    for (size_t i = 0; i < n; ++i) {
        const v3 a = sub(at(tris + 9 * i), c), b = sub(at(tris + 9 * i + 3), c), e = sub(at(tris + 9 * i + 6), c);
        /* std::max({a, b, e, r2}): keeps the first element unless a later one compares greater */
        float m = dot(a, a);
        if (m < dot(b, b)) m = dot(b, b);
        if (m < dot(e, e)) m = dot(e, e);
        if (m < r2) m = r2;
        r2 = m;
    }
    out[0] = c.x;
    out[1] = c.y;
    out[2] = c.z;
    out[3] = sqrtf(r2);
}

/* Mesh::intersects_with_bounding_sphere, mesh.cpp:249-266 */
static int sphere_hit(const float* sphere, v3 o, v3 d) {
    const v3 oc = sub(o, at(sphere));
    const float b = dot(oc, d);
    const float c = dot(oc, oc) - (sphere[3] * sphere[3]);
    if (c > 0.0f && b > 0.0f) return 0;
    /* volatile: GCC -O3 otherwise folds this test to "true" whenever !(c > 0), which also admits a NaN c (a
     * mesh with a NaN vertex); as written, a NaN discriminant is a miss */
    volatile float discr = (b * b) - c;
    return discr >= 0.0f;
}

static int cmp_float(const void* a, const void* b) {
    const float x = *(const float*)a, y = *(const float*)b;
    return (x > y) - (x < y);
}

/* Mesh::closest_and_farthest_intersections + intersection_distances, mesh.cpp:269-294: the multiset of the
 * distances > 0, then its ends.  scratch: n floats.  Returns 1 with bounds[0..1] set, else 0. */
static int closest_and_farthest(const float* tris, size_t n, const float* sphere, const float* offset,
                                const float* direction, float* scratch, float* bounds) {
    if (!sphere_hit(sphere, at(offset), at(direction))) return 0;
    size_t m = 0;
    for (size_t i = 0; i < n; ++i) {
        const float t = orc_tri_intersect(tris + 9 * i, offset, direction);
        if (t > 0) scratch[m++] = t;
    }
    if (m == 0) return 0;
    qsort(scratch, m, sizeof(float), cmp_float);
    bounds[0] = m > 1 ? scratch[0] : 0.0f;
    bounds[1] = scratch[m - 1];
    return 1;
}

int orc_closest_and_farthest(const float* tris, size_t n, const float* offset, const float* direction,
                             float* bounds) {
    float sphere[4];
    orc_bounding_sphere(tris, n, sphere);
    float* scratch = (float*)malloc((n ? n : 1) * sizeof(float));
    const int r = closest_and_farthest(tris, n, sphere, offset, direction, scratch, bounds);
    free(scratch);
    return r;
}

/* Zone::render's loop, zone.cpp:101-134, over one LUT (direction / offset: rows*cols x 3 doubles).
 * Returns 0, -1 for "Zone::render: range overflow", -2 for the area error; *pixels gets
 * pixels_with_intersections. */
int orc_zone_render(const float* tris, size_t n, const double* direction, const double* offset, size_t rows,
                    size_t cols, uint32_t point_count, uint32_t* near_mm, uint32_t* far_mm, uint32_t* pixels) {
    float sphere[4];
    orc_bounding_sphere(tris, n, sphere);
    float* scratch = (float*)malloc((n ? n : 1) * sizeof(float));
    uint32_t hits = 0;
    for (size_t row = 0; row < rows; ++row)
        for (size_t col = 0; col < cols; ++col) {
            const size_t p = row * cols + col;
            const float o[3] = {(float)offset[3 * p], (float)offset[3 * p + 1], (float)offset[3 * p + 2]};
            const float d[3] = {(float)direction[3 * p] * 1000.0f, (float)direction[3 * p + 1] * 1000.0f,
                                (float)direction[3 * p + 2] * 1000.0f};
            float bounds[2];
            if (closest_and_farthest(tris, n, sphere, o, d, scratch, bounds))
                hits++;
            else
                bounds[0] = bounds[1] = 0.f;
            const double nm = round(bounds[0] * 1000.0), fm = round(bounds[1] * 1000.0);
            if (nm > UINT32_MAX || fm > UINT32_MAX) {
                free(scratch);
                *pixels = hits;
                return -1;
            }
            near_mm[p] = (uint32_t)nm;
            far_mm[p] = (uint32_t)fm;
        }
    free(scratch);
    *pixels = hits;
    if (hits > 0 && hits < point_count) return -2;
    return 0;
}

/* EmulatedZoneMon._calc_counts for one live zone, python/src/ouster/sdk/core/zone_common.py:47-78.
 * out: count, occlusion, invalid, min, max, mean (numpy's float64 mean truncated into uint32; 0 when empty).
 * bitmask (optional) gets 1 << live_index OR-ed where the zone triggers. */
void orc_zone_counts(const uint32_t* range, const uint32_t* near_mm, const uint32_t* far_mm, size_t npx,
                     uint32_t live_index, uint32_t* bitmask, uint32_t* out) {
    uint32_t count = 0, occlusion = 0, invalid = 0, mn = UINT32_MAX, mx = 0;
    uint64_t sum = 0;
    for (size_t p = 0; p < npx; ++p) {
        const uint32_t r = range[p];
        const int trig = r > 0 && near_mm[p] <= r && r <= far_mm[p];
        if (trig) {
            count++;
            sum += r;
            if (r < mn) mn = r;
            if (r > mx) mx = r;
            if (bitmask) bitmask[p] |= 1u << live_index;
        }
        invalid += r == 0 && near_mm[p] > 0;
        occlusion += r > 0 && r <= near_mm[p];
    }
    out[0] = count;
    out[1] = occlusion;
    out[2] = invalid;
    out[3] = count ? mn : 0;
    out[4] = count ? mx : 0;
    out[5] = count ? (uint32_t)((double)sum / (double)count) : 0;
}

/* calc_triggers' counters for one live zone, zone_common.py:86-105.  mode: 1 OCCUPANCY, 2 VACANCY. */
void orc_zone_trigger(int mode, uint32_t point_count, uint32_t frame_count, uint32_t count, uint32_t* triggers,
                      uint32_t* alerts) {
    if ((count >= point_count && mode == 1) || (count < point_count && mode == 2))
        *triggers += 1;
    else
        *triggers = 0;
    if (*triggers >= frame_count)
        *alerts += 1;
    else
        *alerts = 0;
}
