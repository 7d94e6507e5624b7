/*
 * orc_icp.c -- CPU oracle for frame-to-map registration (DESIGN f-6): VoxelHashMap3d and ICP.
 *
 * TEST INFRASTRUCTURE ONLY (like the rest of oracle/, see ouster_oracle.h).  Plain-C restatement of
 *   ouster_core/src/voxel_hash_map.cpp:14-41           VoxelHashMap constructor checks, map_resolution_sq
 *   ouster_core/src/voxel_hash_map.cpp:85-107          add_point / add_points
 *   ouster_core/include/ouster/core/voxel_hash_map.h:287-301   first_n_point
 *   ouster_core/src/voxel_hash_map.cpp:109-154         remove_ / extract_voxels_far_from_location
 *   ouster_core/src/voxel_hash_map.cpp:43-76           pointcloud
 *   ouster_core/src/voxel_hash_map.cpp:159-247         VOXEL_SHIFTS, get_closest_neighbor
 *   ouster_mapping/src/icp_registration.cpp            data_association, build_linear_system, align_points_to_map
 *   thirdparty/sophus/sophus/so3.hpp:344-397, 527-534, 550-571, 694-731   SO3 product / action / normalise,
 *                                                      leftJacobian, expAndTheta
 *   thirdparty/sophus/sophus/se3.hpp:273-322, 852-861  SE3 matrix, product, action, exp
 *   Eigen LDLT (ldlt_inplace<Lower>::unblocked, LDLT::_solve_impl), inner products summed in index order
 * (all paths relative to the reference tree, ouster-sdk 1.0.1).
 *
 * Order: voxels are kept in an array in creation order; pointcloud() and the extracted rows come out in that order,
 * inside a voxel in slot order (the reference: tsl::robin_map order, DESIGN 9).
 * Integer voxel distances wrap in int32 as the reference compiles on x86 (computed here in uint32, no UB).
 * -ffp-contract=off keeps every product and sum rounded on its own.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int32_t k[3];
    int alive;
    size_t cnt;
} orc_voxel;

typedef struct {
    double voxel_size, max_distance, inv, res_sq;
    size_t max_pts, min_pts;
    orc_voxel* vox; /* creation order */
    double* pts;    /* n_vox x max_pts x 3 */
    size_t n_vox, cap_vox, live, points;
    int64_t* index; /* open addressing voxel -> vox id; -1 empty, -2 erased */
    size_t icap, iused;
} orc_map;

/* Returns 0 and *out, or -1 "max_points_per_voxel must be greater than 0", -2 "voxel_size must be greater than 0",
 * -3 "max_distance must be greater than 0", in the reference's order. */
int orc_map_create(double voxel_size, double max_distance, size_t max_pts, size_t min_pts, orc_map** out);
void orc_map_destroy(orc_map* m);
void orc_map_clear(orc_map* m);
void orc_map_add_points(orc_map* m, const double* p, size_t n);
size_t orc_map_remove_far(orc_map* m, const double* origin, double* extracted);
size_t orc_map_size(const orc_map* m, size_t* points);
size_t orc_map_point_cloud(const orc_map* m, double* out);
double orc_map_closest(const orc_map* m, const double* q, double max_d2, double* nb);
void orc_linear_system(const double* src, const double* tgt, size_t n, double ks, double* jtj, double* jtr);
void orc_ldlt_solve6(const double* A, const double* b, double* x);
void orc_se3_exp(const double* a, double* M);
int orc_icp_align(const orc_map* m, const double* frame, size_t n, double max_distance, double kernel_scale,
                  int max_iterations, double criterion, double* M);
int32_t orc_cull_threshold(double max_distance, double voxel_size);

static int32_t voxel_coord(double v) {
    const double f = floor(v);
    if (!(f >= -2147483648.0 && f < 2147483648.0)) return INT32_MIN;
    return (int32_t)f;
}

static double sqn3(double a, double b, double c) { return (a * a + b * b) + c * c; }

static size_t khash(const int32_t* k, size_t mask) {
    uint64_t h = (uint64_t)(uint32_t)k[0] * 0x9E3779B97F4A7C15ull;
    h ^= (uint64_t)(uint32_t)k[1] * 0xC2B2AE3D27D4EB4Full;
    h ^= (uint64_t)(uint32_t)k[2] * 0x165667B19E3779F9ull;
    h ^= h >> 29;
    return (size_t)h & mask;
}

static void index_rebuild(orc_map* m, size_t want) {
    size_t cap = 64;
    while (cap < 2 * want + 64) cap <<= 1;
    free(m->index);
    m->index = (int64_t*)malloc(cap * sizeof(int64_t));
    if (!m->index) abort();
    memset(m->index, 0xff, cap * sizeof(int64_t));
    m->icap = cap;
    m->iused = 0;
    for (size_t v = 0; v < m->n_vox; ++v) {
        if (!m->vox[v].alive) continue;
        size_t i = khash(m->vox[v].k, cap - 1);
        while (m->index[i] != -1) i = (i + 1) & (cap - 1);
        m->index[i] = (int64_t)v;
        m->iused++;
    }
}

/* index slot holding voxel k, or the -1 slot that ends its probe chain */
static size_t index_find(const orc_map* m, const int32_t* k) {
    size_t i = khash(k, m->icap - 1);
    for (;;) {
        const int64_t v = m->index[i];
        if (v == -1) return i;
        if (v >= 0 && memcmp(m->vox[v].k, k, sizeof(int32_t) * 3) == 0) return i;
        i = (i + 1) & (m->icap - 1);
    }
}

int orc_map_create(double voxel_size, double max_distance, size_t max_pts, size_t min_pts, orc_map** out) {
    if (max_pts == 0) return -1;
    if (voxel_size <= 0) return -2;
    if (max_distance <= 0) return -3;
    orc_map* m = (orc_map*)calloc(1, sizeof(orc_map));
    if (!m) abort();
    m->voxel_size = voxel_size;
    m->max_distance = max_distance;
    m->max_pts = max_pts;
    m->min_pts = min_pts;
    m->res_sq = voxel_size * voxel_size / (double)max_pts;
    m->inv = 1.0 / voxel_size;
    index_rebuild(m, 0);
    *out = m;
    return 0;
}

void orc_map_destroy(orc_map* m) {
    if (!m) return;
    free(m->vox);
    free(m->pts);
    free(m->index);
    free(m);
}

void orc_map_clear(orc_map* m) {
    m->n_vox = m->live = m->points = 0;
    index_rebuild(m, 0);
}

static void voxel_of(const orc_map* m, const double* p, int32_t* k) {
    k[0] = voxel_coord(p[0] * m->inv);
    k[1] = voxel_coord(p[1] * m->inv);
    k[2] = voxel_coord(p[2] * m->inv);
}

/* add_point (voxel_hash_map.cpp:85-99) with first_n_point (voxel_hash_map.h:287-301) */
static void add_point(orc_map* m, const double* p) {
    int32_t k[3];
    voxel_of(m, p, k);
    size_t i = index_find(m, k);
    int64_t v = m->index[i];
    if (v < 0) {
        if (2 * (m->iused + 1) > m->icap) {
            index_rebuild(m, m->live + 1);
            i = index_find(m, k);
        }
        if (m->n_vox == m->cap_vox) {
            m->cap_vox = m->cap_vox ? 2 * m->cap_vox : 256;
            m->vox = (orc_voxel*)realloc(m->vox, m->cap_vox * sizeof(orc_voxel));
            m->pts = (double*)realloc(m->pts, m->cap_vox * m->max_pts * 3 * sizeof(double));
            if (!m->vox || !m->pts) abort();
        }
        v = (int64_t)m->n_vox++;
        memcpy(m->vox[v].k, k, sizeof(k));
        m->vox[v].alive = 1;
        m->vox[v].cnt = 0;
        m->index[i] = v;
        m->iused++;
        m->live++;
    }
    orc_voxel* b = &m->vox[v];
    double* bp = m->pts + (size_t)v * m->max_pts * 3;
    if (b->cnt == m->max_pts) return;
    for (size_t j = 0; j < b->cnt; ++j)
        if (sqn3(bp[3 * j] - p[0], bp[3 * j + 1] - p[1], bp[3 * j + 2] - p[2]) < m->res_sq) return;
    memcpy(bp + 3 * b->cnt, p, 3 * sizeof(double));
    b->cnt++;
    m->points++;
}

void orc_map_add_points(orc_map* m, const double* p, size_t n) {
    for (size_t i = 0; i < n; ++i) add_point(m, p + 3 * i);
}

int32_t orc_cull_threshold(double max_distance, double voxel_size) {
    const double c = ceil(max_distance * (1.0 / voxel_size));
    const uint32_t d = (uint32_t)voxel_coord(c) + 1u;
    return (int32_t)(d * d);
}

/* remove_voxels_far_from_location / extract_voxels_far_from_location (voxel_hash_map.cpp:109-154); extracted may be
 * NULL; returns the number of extracted rows */
size_t orc_map_remove_far(orc_map* m, const double* origin, double* extracted) {
    int32_t o[3];
    voxel_of(m, origin, o);
    const int32_t thr = orc_cull_threshold(m->max_distance, m->voxel_size);
    size_t rows = 0;
    for (size_t v = 0; v < m->n_vox; ++v) {
        orc_voxel* b = &m->vox[v];
        if (!b->alive) continue;
        const uint32_t dx = (uint32_t)b->k[0] - (uint32_t)o[0], dy = (uint32_t)b->k[1] - (uint32_t)o[1],
                       dz = (uint32_t)b->k[2] - (uint32_t)o[2];
        if ((int32_t)((dx * dx + dy * dy) + dz * dz) < thr) continue;
        if (extracted) memcpy(extracted + 3 * rows, m->pts + v * m->max_pts * 3, b->cnt * 3 * sizeof(double));
        rows += b->cnt;
        b->alive = 0;
        m->live--;
        m->points -= b->cnt;
        m->index[index_find(m, b->k)] = -2;
    }
    return rows;
}

size_t orc_map_size(const orc_map* m, size_t* points) {
    if (points) *points = m->points;
    return m->live;
}

size_t orc_map_point_cloud(const orc_map* m, double* out) {
    size_t rows = 0;
    for (size_t v = 0; v < m->n_vox; ++v) {
        if (!m->vox[v].alive) continue;
        memcpy(out + 3 * rows, m->pts + v * m->max_pts * 3, m->vox[v].cnt * 3 * sizeof(double));
        rows += m->vox[v].cnt;
    }
    return rows;
}

static const int8_t SHIFTS[27][3] = {
    {0, 0, 0},   {1, 0, 0},   {-1, 0, 0},  {0, 1, 0},   {0, -1, 0},   {0, 0, 1},  {0, 0, -1},  {1, 1, 0},   {1, -1, 0},
    {-1, 1, 0},  {-1, -1, 0}, {1, 0, 1},   {1, 0, -1},  {-1, 0, 1},   {-1, 0, -1}, {0, 1, 1},  {0, 1, -1},  {0, -1, 1},
    {0, -1, -1}, {1, 1, 1},   {1, 1, -1},  {1, -1, 1},  {1, -1, -1},  {-1, 1, 1}, {-1, 1, -1}, {-1, -1, 1}, {-1, -1, -1},
};

/* get_closest_neighbor (voxel_hash_map.cpp:194-247): returns the squared distance, *nb the point */
double orc_map_closest(const orc_map* m, const double* q, double max_d2, double* nb) {
    int32_t v[3];
    voxel_of(m, q, v);
    double best = max_d2;
    nb[0] = nb[1] = nb[2] = 0.0;
    for (int s = 0; s < 27; ++s) {
        int32_t w[3];
        double lb = 0.0;
        for (int d = 0; d < 3; ++d) {
            w[d] = (int32_t)((uint32_t)v[d] + (uint32_t)(int32_t)SHIFTS[s][d]);
            const double lo = (double)w[d] * m->voxel_size;
            const double hi = lo + m->voxel_size;
            if (q[d] < lo) {
                const double delta = lo - q[d];
                lb += delta * delta;
            } else if (q[d] > hi) {
                const double delta = q[d] - hi;
                lb += delta * delta;
            }
        }
        if (lb >= best) continue;
        const int64_t id = m->index[index_find(m, w)];
        if (id < 0) continue;
        const double* b = m->pts + (size_t)id * m->max_pts * 3;
        for (size_t k = 0; k < m->vox[id].cnt; ++k) {
            const double d2 = sqn3(b[3 * k] - q[0], b[3 * k + 1] - q[1], b[3 * k + 2] - q[2]);
            if (d2 < best) {
                best = d2;
                memcpy(nb, b + 3 * k, 3 * sizeof(double));
            }
        }
    }
    return best;
}

/* ---- build_linear_system with tbb::parallel_deterministic_reduce's tree (grain 128) ---- */
/* jtj entries a pair touches (row, col), then jtr */
static const int JTJ_RC[15][2] = {{0, 0}, {1, 1}, {2, 2}, {3, 1}, {3, 2}, {4, 0}, {4, 2}, {5, 0},
                                  {5, 1}, {3, 3}, {4, 3}, {4, 4}, {5, 3}, {5, 4}, {5, 5}};

static void leaf(const double* src, const double* tgt, size_t b, size_t e, double ks, double* a) {
    memset(a, 0, 21 * sizeof(double));
    for (size_t i = b; i < e; ++i) {
        const double sx = src[3 * i], sy = src[3 * i + 1], sz = src[3 * i + 2];
        const double rx = sx - tgt[3 * i], ry = sy - tgt[3 * i + 1], rz = sz - tgt[3 * i + 2];
        const double kr = ks + sqn3(rx, ry, rz);
        const double w = (ks * ks) / (kr * kr);
        const double wsx = w * sx, wsy = w * sy, wsz = w * sz;
        a[0] += w;
        a[1] += w;
        a[2] += w;
        a[3] -= wsz;
        a[4] += wsy;
        a[5] += wsz;
        a[6] -= wsx;
        a[7] -= wsy;
        a[8] += wsx;
        const double wsx2 = wsx * sx, wsy2 = wsy * sy, wsz2 = wsz * sz;
        a[9] += wsy2 + wsz2;
        a[10] -= wsx * sy;
        a[11] += wsx2 + wsz2;
        a[12] -= wsx * sz;
        a[13] -= wsy * sz;
        a[14] += wsx2 + wsy2;
        a[15] += w * rx;
        a[16] += w * ry;
        a[17] += w * rz;
        const double cx = sy * rz - sz * ry, cy = sz * rx - sx * rz, cz = sx * ry - sy * rx;
        a[18] += w * cx;
        a[19] += w * cy;
        a[20] += w * cz;
    }
}

static void reduce(const double* src, const double* tgt, size_t b, size_t e, double ks, double* a) {
    if (e - b <= 128) {
        leaf(src, tgt, b, e, ks, a);
        return;
    }
    const size_t mid = b + (e - b) / 2;
    double r[21];
    reduce(src, tgt, b, mid, ks, a);
    reduce(src, tgt, mid, e, ks, r);
    for (int j = 0; j < 21; ++j) a[j] = a[j] + r[j];
}

/* jtj: 36 row-major (lower triangle; the rest +0.0), jtr: 6 */
void orc_linear_system(const double* src, const double* tgt, size_t n, double ks, double* jtj, double* jtr) {
    double a[21];
    reduce(src, tgt, 0, n, ks, a);
    memset(jtj, 0, 36 * sizeof(double));
    for (int j = 0; j < 15; ++j) jtj[JTJ_RC[j][0] * 6 + JTJ_RC[j][1]] = a[j];
    for (int j = 0; j < 6; ++j) jtr[j] = a[15 + j];
}

/* ---- Eigen LDLT on the lower triangle: diagonal pivoting (largest |d|, first on ties), pivots of |d| <= DBL_MIN
 * give a zero solution component ---- */
void orc_ldlt_solve6(const double* A, const double* rhs, double* x) {
    double m[6][6];
    int tr[6];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) m[i][j] = j <= i ? A[i * 6 + j] : 0.0;
    for (int k = 0; k < 6; ++k) {
        int big = k;
        double bv = fabs(m[k][k]);
        for (int i = k + 1; i < 6; ++i)
            if (fabs(m[i][i]) > bv) {
                bv = fabs(m[i][i]);
                big = i;
            }
        tr[k] = big;
        if (k != big) {
            double s;
            for (int j = 0; j < k; ++j) {
                s = m[k][j];
                m[k][j] = m[big][j];
                m[big][j] = s;
            }
            for (int i = big + 1; i < 6; ++i) {
                s = m[i][k];
                m[i][k] = m[i][big];
                m[i][big] = s;
            }
            s = m[k][k];
            m[k][k] = m[big][big];
            m[big][big] = s;
            for (int i = k + 1; i < big; ++i) {
                s = m[i][k];
                m[i][k] = m[big][i];
                m[big][i] = s;
            }
        }
        if (k > 0) {
            double temp[6];
            for (int j = 0; j < k; ++j) temp[j] = m[j][j] * m[k][j];
            double dot = m[k][0] * temp[0];
            for (int j = 1; j < k; ++j) dot = dot + m[k][j] * temp[j];
            m[k][k] = m[k][k] - dot;
            for (int i = k + 1; i < 6; ++i) {
                double s = m[i][0] * temp[0];
                for (int j = 1; j < k; ++j) s = s + m[i][j] * temp[j];
                m[i][k] = m[i][k] - s;
            }
        }
        const double akk = m[k][k];
        const int valid = fabs(akk) > 0.0;
        if (k == 0 && !valid) { /* the whole diagonal is zero */
            for (int j = 0; j < 6; ++j) {
                tr[j] = j;
                for (int i = j + 1; i < 6; ++i) m[i][j] = 0.0;
            }
            break;
        }
        if (valid)
            for (int i = k + 1; i < 6; ++i) m[i][k] = m[i][k] / akk;
    }
    for (int i = 0; i < 6; ++i) x[i] = rhs[i];
    for (int k = 0; k < 6; ++k) {
        const double s = x[k];
        x[k] = x[tr[k]];
        x[tr[k]] = s;
    }
    for (int j = 0; j < 6; ++j)
        for (int i = j + 1; i < 6; ++i) x[i] = x[i] - x[j] * m[i][j];
    for (int i = 0; i < 6; ++i) x[i] = fabs(m[i][i]) > DBL_MIN ? x[i] / m[i][i] : 0.0;
    for (int i = 4; i >= 0; --i) {
        double s = m[i + 1][i] * x[i + 1];
        for (int j = i + 2; j < 6; ++j) s = s + m[j][i] * x[j];
        x[i] = x[i] - s;
    }
    for (int k = 5; k >= 0; --k) {
        const double s = x[k];
        x[k] = x[tr[k]];
        x[tr[k]] = s;
    }
}

/* ---- Sophus ---- */
typedef struct {
    double q[4]; /* x, y, z, w */
    double t[3];
} se3;

static void cross3(const double* a, const double* b, double* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}
static void rotate(const double* q, const double* p, double* out) {
    double uv[3], c[3];
    cross3(q, p, uv);
    for (int d = 0; d < 3; ++d) uv[d] = uv[d] + uv[d];
    cross3(q, uv, c);
    for (int d = 0; d < 3; ++d) out[d] = (p[d] + q[3] * uv[d]) + c[d];
}
static void se3_apply(const se3* g, const double* p, double* out) {
    double r[3];
    rotate(g->q, p, r);
    for (int d = 0; d < 3; ++d) out[d] = r[d] + g->t[d];
}
static se3 se3_mul(const se3* a, const se3* b) {
    se3 c;
    const double ax = a->q[0], ay = a->q[1], az = a->q[2], aw = a->q[3];
    const double bx = b->q[0], by = b->q[1], bz = b->q[2], bw = b->q[3];
    c.q[3] = aw * bw - ax * bx - ay * by - az * bz;
    c.q[0] = aw * bx + ax * bw + ay * bz - az * by;
    c.q[1] = aw * by + ay * bw + az * bx - ax * bz;
    c.q[2] = aw * bz + az * bw + ax * by - ay * bx;
    const double len = sqrt((c.q[0] * c.q[0] + c.q[2] * c.q[2]) + (c.q[1] * c.q[1] + c.q[3] * c.q[3]));
    for (int j = 0; j < 4; ++j) c.q[j] = c.q[j] / len;
    double r[3];
    rotate(a->q, b->t, r);
    for (int d = 0; d < 3; ++d) c.t[d] = a->t[d] + r[d];
    return c;
}
static se3 se3_exp(const double* a) {
    const double eps = DBL_EPSILON;
    const double* om = a + 3;
    const double theta_sq = sqn3(om[0], om[1], om[2]);
    double theta, imag, real;
    if (theta_sq < eps * eps) {
        theta = 0.0;
        const double po4 = theta_sq * theta_sq;
        imag = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * po4;
        real = 1.0 - (1.0 / 8.0) * theta_sq + (1.0 / 384.0) * po4;
    } else {
        theta = sqrt(theta_sq);
        const double half = 0.5 * theta;
        imag = sin(half) / theta;
        real = cos(half);
    }
    se3 g;
    g.q[0] = imag * om[0];
    g.q[1] = imag * om[1];
    g.q[2] = imag * om[2];
    g.q[3] = real;
    const double O[3][3] = {{0.0, -om[2], om[1]}, {om[2], 0.0, -om[0]}, {-om[1], om[0], 0.0}};
    double V[3][3];
    const double tsq = theta * theta;
    if (tsq < eps * eps) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) V[i][j] = (i == j ? 1.0 : 0.0) + 0.5 * O[i][j];
    } else {
        const double c1 = (1.0 - cos(theta)) / tsq;
        const double c2 = (theta - sin(theta)) / (tsq * theta);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                const double o2 = (O[i][0] * O[0][j] + O[i][1] * O[1][j]) + O[i][2] * O[2][j];
                V[i][j] = ((i == j ? 1.0 : 0.0) + c1 * O[i][j]) + c2 * o2;
            }
    }
    for (int i = 0; i < 3; ++i) g.t[i] = (V[i][0] * a[0] + V[i][1] * a[1]) + V[i][2] * a[2];
    return g;
}
static void se3_matrix(const se3* g, double* M) {
    const double x = g->q[0], y = g->q[1], z = g->q[2], w = g->q[3];
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    const double R[9] = {1.0 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.0 - (txx + tzz),
                         tyz - twx,         txz - twy, tyz + twx, 1.0 - (txx + tyy)};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) M[i * 4 + j] = R[i * 3 + j];
        M[i * 4 + 3] = g->t[i];
    }
    M[12] = M[13] = M[14] = 0.0;
    M[15] = 1.0;
}

/* SE3::exp(a).matrix(), a = (upsilon, omega) */
void orc_se3_exp(const double* a, double* M) {
    const se3 g = se3_exp(a);
    se3_matrix(&g, M);
}

/* align_points_to_map_impl (icp_registration.cpp); returns the iterations run, M = t_icp.matrix() */
int orc_icp_align(const orc_map* m, const double* frame, size_t n, double max_distance, double kernel_scale,
                  int max_iterations, double criterion, double* M) {
    se3 pose = {{0.0, 0.0, 0.0, 1.0}, {0.0, 0.0, 0.0}};
    if (m->live == 0) {
        se3_matrix(&pose, M);
        return 0;
    }
    double* src = (double*)malloc((n ? n : 1) * 3 * sizeof(double));
    double* ps = (double*)malloc((n ? n : 1) * 3 * sizeof(double));
    double* pt = (double*)malloc((n ? n : 1) * 3 * sizeof(double));
    if (!src || !ps || !pt) abort();
    memcpy(src, frame, n * 3 * sizeof(double));
    const double md2 = max_distance * max_distance;
    int it = 0;
    while (it < max_iterations) {
        size_t np = 0;
        for (size_t i = 0; i < n; ++i) { /* data_association, compacted in source order */
            double nb[3];
            if (orc_map_closest(m, src + 3 * i, md2, nb) < md2) {
                memcpy(ps + 3 * np, src + 3 * i, 3 * sizeof(double));
                memcpy(pt + 3 * np, nb, 3 * sizeof(double));
                ++np;
            }
        }
        double jtj[36], jtr[6], rhs[6], dx[6];
        orc_linear_system(ps, pt, np, kernel_scale, jtj, jtr);
        for (int j = 0; j < 6; ++j) rhs[j] = -jtr[j];
        orc_ldlt_solve6(jtj, rhs, dx);
        const se3 est = se3_exp(dx);
        for (size_t i = 0; i < n; ++i) {
            double q[3];
            se3_apply(&est, src + 3 * i, q);
            memcpy(src + 3 * i, q, sizeof(q));
        }
        pose = se3_mul(&est, &pose);
        ++it;
        /* Vector6d::squaredNorm in Eigen's two-lane order */
        const double sq = (dx[0] * dx[0] + (dx[2] * dx[2] + dx[4] * dx[4])) + (dx[1] * dx[1] + (dx[3] * dx[3] + dx[5] * dx[5]));
        if (sq < criterion * criterion) break;
    }
    se3_matrix(&pose, M);
    free(src);
    free(ps);
    free(pt);
    return it;
}
