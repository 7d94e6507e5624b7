/*
 * orc_normals.c -- CPU oracle for surface normals on destaggered XYZ (SURVEY 8f-2).
 *
 * TEST INFRASTRUCTURE ONLY (see ouster_oracle.h).  Plain-C restatement of
 *   ouster_algorithm/src/normals.cpp:32-76   compute_vertical_subtent
 *   ouster_algorithm/src/normals.cpp:78-407  compute_unit_normals
 *   ouster_algorithm/src/normals.cpp:411-483 the two public overloads
 * (all paths relative to /root/reference, ouster-sdk 1.0.1).
 *
 * Floating point: double throughout, one rounding per operation (-ffp-contract=off).  The 3-term
 * reductions (dot, squaredNorm) are summed as (x0 + x1) + x2 -- Eigen 3.4's unrolled SSE2 redux for
 * fixed-size 3-vectors (one 2-wide packet, then the scalar tail); the reference's own tests pin this
 * path to np.allclose on hand-computed values only (python/tests/test_normals.py:362-442), so the
 * summation order is a documented choice, not a pinned fact.
 *
 * Parity status: pinned to those known answers (tests/test_oracle_normals.py); everything else is
 * checked through properties (unit length, planar scenes).
 */
#define _GNU_SOURCE
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ouster_oracle.h"

#define FOREGROUND_SALIENCE_MM 500 /* normals.cpp:24 */

static double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static double sqn3(const double* a) { return dot3(a, a); }

/* normalized beam of pixel (row, col): xyz minus the column's sensor origin, divided by its norm
 * (normals.cpp:111-129); zero vector when the magnitude is zero */
static void beam_of(const double* xyz, const double* origins, size_t w, size_t row, size_t col, double* out) {
    const double* p = xyz + (row * w + col) * 3;
    double d[3] = {p[0], p[1], p[2]};
    if (origins) {
        d[0] -= origins[col * 3 + 0];
        d[1] -= origins[col * 3 + 1];
        d[2] -= origins[col * 3 + 2];
    }
    const double mag = sqrt(sqn3(d));
    if (mag > 0.0) {
        out[0] = d[0] / mag;
        out[1] = d[1] / mag;
        out[2] = d[2] / mag;
    } else {
        out[0] = out[1] = out[2] = 0.0;
    }
}

/* normals.cpp:32-76 */
double orc_normals_vertical_subtent(const double* xyz, const uint32_t* range, const double* origins,
                                    size_t h, size_t w) {
    const size_t mid_col = w / 2;
    for (size_t col_offset = 0; col_offset <= mid_col; ++col_offset) {
        for (int si = 0; si < 2; ++si) {
            const int sign = si == 0 ? -1 : 1;
            const int col_i = (int)mid_col + sign * (int)col_offset;
            if (col_i < 0 || col_i >= (int)w) continue;
            const size_t col = (size_t)col_i;
            size_t top = h > 0 ? h - 1 : 0;
            size_t bottom = 0;
            while (top > bottom) {
                const int ht = range[top * w + col] != 0, hb = range[bottom * w + col] != 0;
                if (ht && hb) {
                    double vt[3], vb[3];
                    beam_of(xyz, origins, w, top, col, vt);
                    beam_of(xyz, origins, w, bottom, col, vb);
                    double dp = dot3(vt, vb);
                    dp = fmax(-1.0, fmin(1.0, dp));
                    const double angle = acos(dp);
                    if (top != bottom) return angle / (double)(top - bottom);
                }
                top -= ht ? 0 : 1;
                bottom += hb ? 0 : 1;
            }
        }
    }
    const size_t intervals = h - 1 > 1 ? h - 1 : 1; /* std::max<size_t>(1, height - 1), size_t arithmetic */
    return (0.5 * M_PI) / (double)intervals;
}

typedef struct {
    const double *xyz, *xyz2;
    const uint32_t *range, *range2;
    size_t h, w;
    double desired_sq;
} nctx;

typedef struct {
    double best_diff[3];
    double min_distance_sq;
    size_t best_radius;
    int best_flip;
    int thin; /* thin_foreground_flag (in/out) */
} nstate;

/* consider_neighbor -- normals.cpp:177-205 */
static void consider(const nctx* c, nstate* s, size_t row, size_t col, const double* xyz_base,
                     const uint32_t* rng_base, int flip, size_t radius, const double* center,
                     uint32_t center_range) {
    const size_t idx = row * c->w + col;
    const uint32_t nr = rng_base[idx];
    if (nr == 0) return;
    const double* nv = xyz_base + idx * 3;
    const double diff[3] = {nv[0] - center[0], nv[1] - center[1], nv[2] - center[2]};
    const double dsq = sqn3(diff);
    if ((int64_t)nr - (int64_t)center_range < (int64_t)FOREGROUND_SALIENCE_MM) s->thin = 0;
    const double cand = fabs(dsq - c->desired_sq);
    if (cand < fabs(s->min_distance_sq - c->desired_sq)) {
        s->best_diff[0] = diff[0];
        s->best_diff[1] = diff[1];
        s->best_diff[2] = diff[2];
        s->min_distance_sq = dsq;
        s->best_flip = flip;
        s->best_radius = radius;
    }
}

/* find_best_neighbor -- normals.cpp:157-268; vertical != 0: VERTICAL axis */
static int find_best(const nctx* c, int vertical, size_t row, size_t col, double neighbor_sq,
                     const double* center, uint32_t center_range, double* diff, int* flip, int* thin,
                     size_t max_up, size_t max_down, size_t search) {
    nstate s;
    s.best_diff[0] = s.best_diff[1] = s.best_diff[2] = 0.0;
    s.min_distance_sq = INFINITY;
    s.best_radius = 1;
    s.best_flip = 0;
    s.thin = *thin;
    int good = 0;
    const int dual = c->xyz2 != NULL && c->range2 != NULL;
    for (size_t radius = 1; radius <= search; ++radius) {
        if (vertical && radius > max_up && radius > max_down) break;
        if (good && !s.thin) break;
        if (vertical) {
            if (radius <= max_up) consider(c, &s, row - radius, col, c->xyz, c->range, 1, radius, center, center_range);
            if (radius <= max_down) consider(c, &s, row + radius, col, c->xyz, c->range, 0, radius, center, center_range);
            if (dual) {
                if (radius <= max_up) consider(c, &s, row - radius, col, c->xyz2, c->range2, 1, radius, center, center_range);
                if (radius <= max_down) consider(c, &s, row + radius, col, c->xyz2, c->range2, 0, radius, center, center_range);
            }
        } else {
            const int wi = (int)c->w;
            const int lu = (int)col - (int)radius;
            const size_t left = (size_t)(((lu % wi) + wi) % wi);
            consider(c, &s, row, left, c->xyz, c->range, 1, radius, center, center_range);
            if (dual) consider(c, &s, row, left, c->xyz2, c->range2, 1, radius, center, center_range);
            const size_t right = (size_t)(((int)col + (int)radius) % wi);
            consider(c, &s, row, right, c->xyz, c->range, 0, radius, center, center_range);
            if (dual) consider(c, &s, row, right, c->xyz2, c->range2, 0, radius, center, center_range);
        }
        const double lim = (double)s.best_radius * (double)s.best_radius * neighbor_sq;
        if (c->desired_sq <= s.min_distance_sq && s.min_distance_sq < lim) {
            good = 1;
        } else if (radius == search) {
            if (s.min_distance_sq > 0 && s.min_distance_sq < lim) good = 1;
        }
    }
    *thin = s.thin;
    if (good && s.min_distance_sq < INFINITY) {
        diff[0] = s.best_diff[0];
        diff[1] = s.best_diff[1];
        diff[2] = s.best_diff[2];
        *flip = s.best_flip;
        return 1;
    }
    return 0;
}

/* compute_unit_normals -- normals.cpp:78-407.  xyz2/range2 may be NULL.  subtent_override <= 0:
 * computed from (xyz, range).  Returns 0, or -1 "normals: target_distance_m must be positive",
 * -2 "normals: min_angle_of_incidence_rad must be positive". */
int orc_normals_compute(const double* xyz, const uint32_t* range, const double* xyz2,
                        const uint32_t* range2, size_t h, size_t w, const double* origins,
                        double* normals, size_t search, double min_aoi_rad, double target_m,
                        double subtent_override) {
    if (target_m <= 0.0) return -1;
    if (min_aoi_rad <= 0.0) return -2;
    const double h_subtent = 2.0 * M_PI / (double)w;
    const double safe = fmax(min_aoi_rad, 1e-6);
    const double v_subtent = subtent_override > 0.0 ? subtent_override
                                                    : orc_normals_vertical_subtent(xyz, range, origins, h, w);
    nctx c = {xyz, xyz2, range, range2, h, w, target_m * target_m};
    const double tan_safe = tan(safe);
    for (size_t u = 0; u < h; ++u) {
        const size_t max_up = search < u ? search : u;
        const size_t max_down = search < h - 1 - u ? search : h - 1 - u;
        for (size_t v = 0; v < w; ++v) {
            double* n = normals + (u * w + v) * 3;
            n[0] = n[1] = n[2] = 0.0;
            const uint32_t cr = range[u * w + v];
            if (cr == 0) continue;
            const double* center = xyz + (u * w + v) * 3;
            double beam[3];
            beam_of(xyz, origins, w, u, v, beam);
            if (sqn3(beam) <= 2.220446049250313e-16) continue;
            /* calc_max_distance_threshold -- normals.cpp:143-151 */
            const double perimeter = 2.0 * M_PI * ((double)cr * 0.001);
            const double nh = (perimeter / ((2.0 * M_PI) / h_subtent)) / tan_safe;
            const double nv = (perimeter / ((2.0 * M_PI) / v_subtent)) / tan_safe;
            double vd[3] = {0, 0, 0}, hd[3] = {0, 0, 0};
            int vflip = 0, hflip = 0, vthin = 1, hthin = 1;
            const int vfound = find_best(&c, 1, u, v, nv * nv, center, cr, vd, &vflip, &vthin, max_up, max_down, search);
            const int hfound = find_best(&c, 0, u, v, nh * nh, center, cr, hd, &hflip, &hthin, search, search, search);
            if ((!vfound && !hfound) || (vthin && hthin)) { /* case A */
                n[0] = -beam[0];
                n[1] = -beam[1];
                n[2] = -beam[2];
                continue;
            }
            const double* one = NULL; /* case B */
            if (vfound && (!hfound || hthin)) one = vd;
            else if (hfound && (!vfound || vthin)) one = hd;
            if (one) {
                const double denom = sqn3(one);
                if (fabs(denom) < 2.220446049250313e-16) continue;
                const double s = dot3(one, beam) / denom;
                double pr[3] = {beam[0] - s * one[0], beam[1] - s * one[1], beam[2] - s * one[2]};
                const double nsq = sqn3(pr);
                if (fabs(nsq) < 2.220446049250313e-16) continue;
                const double len = sqrt(nsq);
                n[0] = -(pr[0] / len);
                n[1] = -(pr[1] / len);
                n[2] = -(pr[2] / len);
                continue;
            }
            if (hflip != vflip) { /* case C */
                vd[0] = -vd[0];
                vd[1] = -vd[1];
                vd[2] = -vd[2];
            }
            const double cx = vd[1] * hd[2] - vd[2] * hd[1];
            const double cy = vd[2] * hd[0] - vd[0] * hd[2];
            const double cz = vd[0] * hd[1] - vd[1] * hd[0];
            const double cc[3] = {cx, cy, cz};
            const double mag = sqrt(sqn3(cc));
            if (mag != 0.0) {
                n[0] = cx / mag;
                n[1] = cy / mag;
                n[2] = cz / mag;
            }
        }
    }
    return 0;
}

/* normals(xyz, range, xyz2, range2, origins, ...) -- normals.cpp:432-483: one vertical subtent from
 * the first return, passed to both passes; orc_normals_compute ignores a subtent of 0, so then the
 * second pass derives its own from (xyz2, range2).  n2 / xyz2 / range2 may be NULL (single-return
 * overload, normals.cpp:411-430). */
int orc_normals(const double* xyz, const uint32_t* range, const double* xyz2, const uint32_t* range2,
                size_t h, size_t w, const double* origins, size_t search, double min_aoi_rad,
                double target_m, double subtent_override, double* n1, double* n2) {
    if (!xyz2 || !range2)
        return orc_normals_compute(xyz, range, NULL, NULL, h, w, origins, n1, search, min_aoi_rad, target_m,
                                   subtent_override);
    const double sub = subtent_override > 0.0 ? subtent_override
                                              : orc_normals_vertical_subtent(xyz, range, origins, h, w);
    int rc = orc_normals_compute(xyz, range, xyz2, range2, h, w, origins, n1, search, min_aoi_rad, target_m, sub);
    if (rc != 0) return rc;
    return orc_normals_compute(xyz2, range2, xyz, range, h, w, origins, n2, search, min_aoi_rad, target_m, sub);
}
