/*
 * orc_voxel.c -- CPU oracle for voxel-grid downsampling (SURVEY 8f-2, the prefilter beside normals).
 *
 * TEST INFRASTRUCTURE ONLY (like the rest of oracle/, see ouster_oracle.h).  Plain-C restatement of
 *   ouster_core/src/voxel_hash_map.cpp:262-310          core::voxel_downsample (shuffle, first-in wins)
 *   ouster_core/src/voxel_hash_map.cpp:312-393          core::voxel_downsample_3d / _xd
 *   ouster_core/src/voxel_hash_map.cpp:15-41            VoxelHashMap constructor checks, map_resolution_sq
 *   ouster_core/include/ouster/core/voxel_hash_map.h:287-334, 587-635   insertion strategies
 *   ouster_core/include/ouster/core/voxel_hash_map.h:142-185            PointNormalBucket
 *   ouster_algorithm/src/voxel_downsample.cpp:21-57     algorithm::voxel_downsample_with_normals
 * (all paths relative to the reference tree, ouster-sdk 1.0.1).
 *
 * Output order: voxels in the order of their first point in the (possibly shuffled) input, inside a
 * voxel the bucket's slot order.  For orc_voxel_downsample that IS the reference's order; for the other
 * three the reference emits in tsl::robin_map iteration order, which is not reproduced (DESIGN 9).
 *
 * Voxel of a point: floor(p * (1.0 / voxel_size)) cast to int the way x86 cvttsd2si does it -- NaN and
 * values outside [-2^31, 2^31) give INT32_MIN -- written out explicitly (no UB here).
 * squaredNorm / norm of a 3-vector: (x0*x0 + x1*x1) + x2*x2, the association orc_normals.c uses
 * (DESIGN 2); -ffp-contract=off keeps every product and sum rounded on its own.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* Built on its own into libouster_oracle_voxel.so (oracle/voxel.mk) and bound by oracle/voxel.py.
 * orc_voxel_downsample_xd returns 0, -1 "max_points_per_voxel must be greater than 0", -2 "voxel_size must be
 * greater than 0", -3 "frame must have at least 3 columns", -4 "unknown strategy";
 * orc_voxel_downsample_with_normals returns 0 or -1 "voxel_size must be > 0". */
int32_t orc_voxel_coord(double v);
size_t orc_voxel_downsample(const double* frame, size_t n, double voxel_size, double* out, uint32_t* idx_out);
int orc_voxel_downsample_xd(const double* frame, size_t n, size_t cols, double voxel_size, size_t max_pts,
                            size_t min_pts, int strategy, double* out, uint32_t* idx_out, size_t* n_out);
int orc_voxel_downsample_with_normals(const double* pts, const double* nrm, size_t n, double voxel_size,
                                      double* out_p, double* out_n, uint32_t* idx_out, size_t* n_out);

int32_t orc_voxel_coord(double v) {
    const double f = floor(v);
    if (!(f >= -2147483648.0 && f < 2147483648.0)) return INT32_MIN;
    return (int32_t)f;
}

static void voxel_of(const double* p, double inv, int32_t* k) {
    k[0] = orc_voxel_coord(p[0] * inv);
    k[1] = orc_voxel_coord(p[1] * inv);
    k[2] = orc_voxel_coord(p[2] * inv);
}

static double sqn3(const double* a) { return (a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]; }

/* xorshift32 of the reference (voxel_hash_map.cpp:274-279, voxel_hash_map.h:607-612) */
static uint32_t xorshift32(uint32_t* s) {
    *s ^= *s << 13;
    *s ^= *s >> 17;
    *s ^= *s << 5;
    return *s;
}

/* open-addressing map voxel key -> voxel id (ids in insertion order) */
typedef struct {
    int32_t* keys; /* cap x 3 */
    int64_t* ids;  /* -1 = empty */
    size_t cap, n;
} vmap;

static int vmap_init(vmap* m, size_t n_points) {
    size_t cap = 16;
    while (cap < 2 * n_points + 16) cap <<= 1;
    m->keys = (int32_t*)malloc(cap * 3 * sizeof(int32_t));
    m->ids = (int64_t*)malloc(cap * sizeof(int64_t));
    m->cap = cap;
    m->n = 0;
    if (!m->keys || !m->ids) return -1;
    memset(m->ids, 0xff, cap * sizeof(int64_t));
    return 0;
}

static void vmap_free(vmap* m) {
    free(m->keys);
    free(m->ids);
}

/* id of voxel k, inserting it when new (*fresh = 1) */
static int64_t vmap_get(vmap* m, const int32_t* k, int* fresh) {
    uint64_t h = (uint64_t)(uint32_t)k[0] * 0x9E3779B97F4A7C15ull;
    h ^= (uint64_t)(uint32_t)k[1] * 0xC2B2AE3D27D4EB4Full;
    h ^= (uint64_t)(uint32_t)k[2] * 0x165667B19E3779F9ull;
    h ^= h >> 29;
    size_t i = (size_t)h & (m->cap - 1);
    for (;;) {
        if (m->ids[i] < 0) {
            memcpy(m->keys + i * 3, k, 3 * sizeof(int32_t));
            m->ids[i] = (int64_t)m->n++;
            *fresh = 1;
            return m->ids[i];
        }
        if (memcmp(m->keys + i * 3, k, 3 * sizeof(int32_t)) == 0) {
            *fresh = 0;
            return m->ids[i];
        }
        i = (i + 1) & (m->cap - 1);
    }
}

/* voxel_hash_map.cpp:262-310: Fisher-Yates with xorshift32 (seed 42) and Lemire's reduction, then the
 * first point of every voxel in shuffled order.  out: n x 3, idx_out: n.  Returns the number kept. */
size_t orc_voxel_downsample(const double* frame, size_t n, double voxel_size, double* out, uint32_t* idx_out) {
    if (n == 0) return 0;
    uint32_t* idx = (uint32_t*)malloc(n * sizeof(uint32_t));
    vmap m;
    if (!idx || vmap_init(&m, n) != 0) abort();
    for (size_t i = 0; i < n; ++i) idx[i] = (uint32_t)i;
    uint32_t state = 42;
    for (size_t i = 0; i + 1 < n; ++i) {
        const size_t j = i + (size_t)(((uint64_t)xorshift32(&state) * (uint64_t)(n - i)) >> 32);
        const uint32_t t = idx[i];
        idx[i] = idx[j];
        idx[j] = t;
    }
    const double inv = 1.0 / voxel_size;
    size_t kept = 0;
    for (size_t i = 0; i < n; ++i) {
        int32_t k[3];
        int fresh;
        voxel_of(frame + (size_t)idx[i] * 3, inv, k);
        vmap_get(&m, k, &fresh);
        if (fresh) {
            memcpy(out + kept * 3, frame + (size_t)idx[i] * 3, 3 * sizeof(double));
            idx_out[kept++] = idx[i];
        }
    }
    vmap_free(&m);
    free(idx);
    return kept;
}

/* voxel_hash_map.cpp:312-393 (VoxelDownsampleStrategy 0 FIRST_N_POINT, 1 AVERAGE_POINT, 2 RANDOM) on an
 * n x cols frame, voxel from columns 0-2.  out: n x cols; idx_out: n source indices (the admitted /
 * surviving point for FIRST_N and RANDOM, the voxel's first point for AVERAGE).  Returns 0 and *n_out, or
 * -1 "max_points_per_voxel must be greater than 0", -2 "voxel_size must be greater than 0",
 * -3 "...: frame must have at least 3 columns", -4 "...: unknown strategy" (checked in the reference's
 * order: empty input first, then columns, strategy, and the map constructor's two checks). */
int orc_voxel_downsample_xd(const double* frame, size_t n, size_t cols, double voxel_size, size_t max_pts,
                            size_t min_pts, int strategy, double* out, uint32_t* idx_out, size_t* n_out) {
    *n_out = 0;
    if (n == 0) return 0;
    if (cols < 3) return -3;
    if (strategy < 0 || strategy > 2) return -4;
    if (max_pts == 0) return -1;
    if (voxel_size <= 0) return -2; /* NaN passes, as in the reference */
    const double inv = 1.0 / voxel_size;
    const double res_sq = voxel_size * voxel_size / (double)max_pts;
    vmap m;
    int64_t* vox = (int64_t*)malloc(n * sizeof(int64_t));
    if (!vox || vmap_init(&m, n) != 0) abort();
    /* pass 1: voxel ids in first-appearance order, point counts */
    for (size_t i = 0; i < n; ++i) {
        int32_t k[3];
        int fresh;
        voxel_of(frame + i * cols, inv, k);
        vox[i] = vmap_get(&m, k, &fresh);
    }
    const size_t nv = m.n;
    size_t* cnt = (size_t*)calloc(nv + 1, sizeof(size_t));
    if (!cnt) abort();
    for (size_t i = 0; i < n; ++i) cnt[vox[i]]++;
    size_t o = 0;
    if (strategy == 1) { /* AVERAGE_POINT: accumulate_strategy + AveragePointBucket (voxel_hash_map.h:96-123, 312-319) */
        double* sum = (double*)calloc(nv * cols, sizeof(double));
        uint32_t* first = (uint32_t*)malloc(nv * sizeof(uint32_t));
        size_t* seen = (size_t*)calloc(nv, sizeof(size_t));
        if (!sum || !first || !seen) abort();
        for (size_t i = 0; i < n; ++i) {
            double* s = sum + (size_t)vox[i] * cols;
            if (seen[vox[i]]++ == 0) first[vox[i]] = (uint32_t)i;
            for (size_t c = 0; c < cols; ++c) s[c] += frame[i * cols + c];
        }
        for (size_t v = 0; v < nv; ++v) {
            if (cnt[v] < min_pts) continue;
            for (size_t c = 0; c < cols; ++c) out[o * cols + c] = sum[v * cols + c] / (double)cnt[v];
            idx_out[o++] = first[v];
        }
        free(sum);
        free(first);
        free(seen);
    } else { /* DefaultVoxelBucket: slots of voxel v at off[v], at most min(count, max) of them */
        size_t* off = (size_t*)malloc((nv + 1) * sizeof(size_t));
        size_t* fill = (size_t*)calloc(nv, sizeof(size_t));
        uint32_t* slot = (uint32_t*)malloc(n * sizeof(uint32_t));
        if (!off || !fill || !slot) abort();
        off[0] = 0;
        for (size_t v = 0; v < nv; ++v) off[v + 1] = off[v] + (cnt[v] < max_pts ? cnt[v] : max_pts);
        uint32_t state = 42; /* random_selection_strategy::rng_state, one stream for the whole map */
        for (size_t i = 0; i < n; ++i) {
            const size_t v = (size_t)vox[i];
            uint32_t* b = slot + off[v];
            if (strategy == 0) { /* first_n_point (voxel_hash_map.h:287-301) */
                if (fill[v] == max_pts) continue;
                const double* p = frame + i * cols;
                int near = 0;
                for (size_t k = 0; k < fill[v] && !near; ++k) {
                    const double* q = frame + (size_t)b[k] * cols;
                    const double d[3] = {q[0] - p[0], q[1] - p[1], q[2] - p[2]};
                    near = sqn3(d) < res_sq;
                }
                if (!near) b[fill[v]++] = (uint32_t)i;
            } else { /* random_selection_strategy, DefaultVoxelBucket path (voxel_hash_map.h:617-628) */
                if (fill[v] < max_pts) {
                    b[fill[v]++] = (uint32_t)i;
                } else {
                    const size_t j = (size_t)(((uint64_t)xorshift32(&state) * (uint64_t)max_pts) >> 32);
                    b[j] = (uint32_t)i;
                }
            }
        }
        for (size_t v = 0; v < nv; ++v)
            for (size_t k = 0; k < fill[v]; ++k) {
                memcpy(out + o * cols, frame + (size_t)slot[off[v] + k] * cols, cols * sizeof(double));
                idx_out[o++] = slot[off[v] + k];
            }
        free(off);
        free(fill);
        free(slot);
    }
    *n_out = o;
    free(cnt);
    free(vox);
    vmap_free(&m);
    return 0;
}

static int finite3(const double* v) { return isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]); }

/* voxel_downsample.cpp:21-57 with PointNormalVoxelHashMap3d (max 1, min 1): rows with a non-finite point
 * or normal, or a normal of norm <= 1e-12, are skipped; the normal is divided by its norm; per voxel the
 * positions are averaged and the unit normals summed and renormalised; a voxel whose normal sum has norm
 * <= 1e-12 is dropped (voxel_hash_map.h:164-175).  idx_out: the voxel's first accepted row.
 * Returns 0, or -1 "voxel_downsample_with_normals voxel_size must be > 0". */
int orc_voxel_downsample_with_normals(const double* pts, const double* nrm, size_t n, double voxel_size,
                                      double* out_p, double* out_n, uint32_t* idx_out, size_t* n_out) {
    *n_out = 0;
    if (!(voxel_size > 0.0)) return -1;
    if (n == 0) return 0;
    const double inv = 1.0 / voxel_size;
    vmap m;
    double* acc = (double*)calloc(n * 6, sizeof(double)); /* per voxel id: point sum, normal sum */
    size_t* cnt = (size_t*)calloc(n, sizeof(size_t));
    uint32_t* first = (uint32_t*)malloc(n * sizeof(uint32_t));
    if (!acc || !cnt || !first || vmap_init(&m, n) != 0) abort();
    for (size_t i = 0; i < n; ++i) {
        const double* p = pts + i * 3;
        const double* q = nrm + i * 3;
        if (!finite3(p) || !finite3(q)) continue;
        const double len = sqrt(sqn3(q));
        if (len <= 1e-12) continue;
        int32_t k[3];
        int fresh;
        voxel_of(p, inv, k);
        const int64_t v = vmap_get(&m, k, &fresh);
        if (fresh) first[v] = (uint32_t)i;
        double* a = acc + (size_t)v * 6;
        for (int c = 0; c < 3; ++c) {
            a[c] += p[c];
            a[3 + c] += q[c] / len;
        }
        cnt[v]++;
    }
    size_t o = 0;
    for (size_t v = 0; v < m.n; ++v) {
        const double* a = acc + v * 6;
        const double len = sqrt(sqn3(a + 3));
        if (len <= 1e-12) continue;
        for (int c = 0; c < 3; ++c) {
            out_p[o * 3 + c] = a[c] / (double)cnt[v];
            out_n[o * 3 + c] = a[3 + c] / len;
        }
        idx_out[o++] = first[v];
    }
    *n_out = o;
    free(acc);
    free(cnt);
    free(first);
    vmap_free(&m);
    return 0;
}
