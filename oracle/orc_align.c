/* orc_align.c -- CPU restatement of cloud-to-cloud ICP (DESIGN f-7).  TEST INFRASTRUCTURE ONLY: nothing under
 * ouster-sdk_b200/ uses it.  Built by oracle/align.mk with the other oracles' flags (-ffp-contract=off: no FMA).
 *
 * What it restates (reference paths relative to the reference tree, ouster-sdk 1.0.1):
 *   median_abs                                   ouster_algorithm/src/align_clouds.cpp:146-161
 *   SpatialHashGrid3D (both constructors, nearest) align_clouds.cpp:170-235
 *   cell of a point, 27-cell order               ouster_algorithm/include/ouster/algorithm/impl/spatial_hash.h:73-101
 *   point_to_point_align                         align_clouds.cpp:1590-1722
 *   point_to_plane_align                         align_clouds.cpp:1724-1874
 *   PoseV::exp (RotV::exp, RotV::vee)            ouster_core/src/transform_vector.cpp:40-60, 96-104
 *   Eigen 3.4 JacobiSVD<Matrix3d> (full U, V), LDLT<Matrix<double, 6, 6>> with info()
 *
 * Evaluation order (DESIGN 2): 3x3 and 4x4 products and matrix-vector products sum over k in index order,
 * ((a0 b0 + a1 b1) + a2 b2) [+ a3 b3]; a 3-vector's squared norm is (x0 x0 + x1 x1) + x2 x2 and its norm the
 * square root of that; dot products as the squared norm.  Sums over correspondences run sequentially in row order,
 * as the reference's loops do.
 *
 * The grid keeps its own hash table (open addressing over the distinct cells); what a lookup returns does not
 * depend on it: the 27 cells are visited in dx, dy, dz order and the rows of a cell in ascending row index. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MIN_ICP_POINTS 20u     /* align_clouds.cpp:308 */
#define MAD_TO_SIGMA 1.4826    /* :310 */
#define HUBER_K 1.5            /* :312 */
#define NORMAL_EPS 1e-12       /* :170 */
#define ICP_MAX_ITERATIONS 10  /* :1600, :1752 */
#define JACOBI_MAX_SWEEPS 64   /* a guard only: a 3x3 converges in a handful of sweeps */

static int finite3(const double* v) { return isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]); }
static double sqn3(double a, double b, double c) { return (a * a + b * b) + c * c; }
static double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static double norm3(const double* a) { return sqrt(sqn3(a[0], a[1], a[2])); }
static double max_d(double a, double b) { return a < b ? b : a; } /* std::max */
static double min_d(double a, double b) { return b < a ? b : a; } /* std::min */

/* static_cast<int64_t>(std::floor(v * inv)) as x86 cvttsd2si evaluates it: NaN and out-of-range give INT64_MIN */
int64_t orc_cell_coord(double v, double inv) {
    const double f = floor(v * inv);
    if (!(f >= -9223372036854775808.0 && f < 9223372036854775808.0)) return INT64_MIN;
    return (int64_t)f;
}

/* ---- median_abs (align_clouds.cpp:146-161): the exact median of |v| ---- */
static int cmp_double(const void* a, const void* b) {
    const double x = *(const double*)a, y = *(const double*)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}
double orc_median_abs(const double* v, size_t n) {
    if (n == 0) return 0.0;
    double* a = malloc(n * sizeof(double));
    for (size_t i = 0; i < n; ++i) a[i] = fabs(v[i]);
    qsort(a, n, sizeof(double), cmp_double);
    const size_t mid = n / 2;
    const double out = (n & 1u) ? a[mid] : 0.5 * (a[mid - 1] + a[mid]);
    free(a);
    return out;
}

/* ---- SpatialHashGrid3D ---- */
typedef struct {
    int64_t c[3];
    int32_t row;
} Entry;
typedef struct {
    double inv;
    size_t n_cells;
    int64_t* keys; /* n_cells x 3 */
    size_t *start, *count;
    int32_t* rows;
    size_t table_cap;
    int64_t* table; /* cell index or -1 */
} Grid;

static int cmp_entry(const void* a, const void* b) {
    const Entry *x = a, *y = b;
    for (int d = 0; d < 3; ++d)
        if (x->c[d] != y->c[d]) return x->c[d] < y->c[d] ? -1 : 1;
    return x->row < y->row ? -1 : (x->row > y->row ? 1 : 0);
}
static uint64_t cell_hash(const int64_t* k) {
    uint64_t h = (uint64_t)k[0] * 0x9E3779B97F4A7C15ull;
    h ^= (uint64_t)k[1] * 0xC2B2AE3D27D4EB4Full;
    h ^= (uint64_t)k[2] * 0x165667B19E3779F9ull;
    h ^= h >> 32;
    h *= 0xD6E8FEB86659FD93ull;
    h ^= h >> 32;
    return h;
}

/* normals == NULL: the point-only constructor (:176-186); otherwise the one that also skips rows whose normal is
 * non-finite or has norm <= NORMAL_EPS (:188-200) */
static void grid_build(Grid* g, const double* pts, const double* normals, size_t m, double cell_size) {
    g->inv = 1.0 / cell_size;
    Entry* e = malloc((m ? m : 1) * sizeof(Entry));
    size_t k = 0;
    for (size_t j = 0; j < m; ++j) {
        const double* p = pts + 3 * j;
        if (!finite3(p)) continue;
        if (normals) {
            const double* nn = normals + 3 * j;
            if (!finite3(nn) || norm3(nn) <= NORMAL_EPS) continue;
        }
        for (int d = 0; d < 3; ++d) e[k].c[d] = orc_cell_coord(p[d], g->inv);
        e[k].row = (int32_t)j;
        ++k;
    }
    qsort(e, k, sizeof(Entry), cmp_entry);
    g->keys = malloc((k ? k : 1) * 3 * sizeof(int64_t));
    g->start = malloc((k ? k : 1) * sizeof(size_t));
    g->count = malloc((k ? k : 1) * sizeof(size_t));
    g->rows = malloc((k ? k : 1) * sizeof(int32_t));
    size_t nc = 0;
    for (size_t i = 0; i < k; ++i) {
        if (i == 0 || memcmp(e[i].c, e[i - 1].c, sizeof(e[i].c)) != 0) {
            memcpy(g->keys + 3 * nc, e[i].c, sizeof(e[i].c));
            g->start[nc] = i;
            g->count[nc] = 0;
            ++nc;
        }
        g->count[nc - 1]++;
        g->rows[i] = e[i].row;
    }
    g->n_cells = nc;
    g->table_cap = 16;
    while (g->table_cap < 2 * nc) g->table_cap <<= 1;
    g->table = malloc(g->table_cap * sizeof(int64_t));
    for (size_t i = 0; i < g->table_cap; ++i) g->table[i] = -1;
    for (size_t c = 0; c < nc; ++c) {
        size_t s = (size_t)cell_hash(g->keys + 3 * c) & (g->table_cap - 1);
        while (g->table[s] >= 0) s = (s + 1) & (g->table_cap - 1);
        g->table[s] = (int64_t)c;
    }
    free(e);
}
static void grid_free(Grid* g) {
    free(g->keys);
    free(g->start);
    free(g->count);
    free(g->rows);
    free(g->table);
}
static int64_t grid_find(const Grid* g, const int64_t* k) {
    size_t s = (size_t)cell_hash(k) & (g->table_cap - 1);
    for (;;) {
        const int64_t c = g->table[s];
        if (c < 0) return -1;
        const int64_t* kc = g->keys + 3 * c;
        if (kc[0] == k[0] && kc[1] == k[1] && kc[2] == k[2]) return c;
        s = (s + 1) & (g->table_cap - 1);
    }
}
/* SpatialHashGrid3D::nearest (:203-226) */
static int grid_nearest(const Grid* g, const double* pts, const double* q, double max_dist_sq) {
    if (!finite3(q) || !isfinite(max_dist_sq) || max_dist_sq <= 0.0) return -1;
    int64_t c[3];
    for (int d = 0; d < 3; ++d) c[d] = orc_cell_coord(q[d], g->inv);
    int best = -1;
    double best_d2 = max_dist_sq;
    for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy)
            for (int dz = -1; dz <= 1; ++dz) {
                /* int64 addition wraps as on x86 */
                const int64_t w[3] = {(int64_t)((uint64_t)c[0] + (uint64_t)(int64_t)dx),
                                      (int64_t)((uint64_t)c[1] + (uint64_t)(int64_t)dy),
                                      (int64_t)((uint64_t)c[2] + (uint64_t)(int64_t)dz)};
                const int64_t cell = grid_find(g, w);
                if (cell < 0) continue;
                for (size_t i = g->start[cell]; i < g->start[cell] + g->count[cell]; ++i) {
                    const int j = g->rows[i];
                    const double* p = pts + 3 * (size_t)j;
                    const double d2 = sqn3(p[0] - q[0], p[1] - q[1], p[2] - q[2]);
                    if (d2 < best_d2) {
                        best_d2 = d2;
                        best = j;
                    }
                }
            }
    return best;
}

/* batch nearest: a grid over the target rows (with the normal filter when normals != NULL) */
void orc_cloud_nearest(const double* tgt, const double* normals, size_t m, double cell_size, const double* queries,
                       size_t nq, double max_dist_sq, int32_t* out) {
    Grid g;
    grid_build(&g, tgt, normals, m, cell_size);
    for (size_t i = 0; i < nq; ++i) out[i] = grid_nearest(&g, tgt, queries + 3 * i, max_dist_sq);
    grid_free(&g);
}

/* ---- Eigen 3.4 JacobiSVD<Matrix3d>(A, ComputeFullU | ComputeFullV) ----
 * No QR preconditioner for a square matrix; two-sided Jacobi sweeps over (p, q) = (1,0), (2,0), (2,1) with
 * real_2x2_jacobi_svd and JacobiRotation::makeJacobi; then |diagonal| with U's column negated for a negative entry,
 * rescaled, and sorted in decreasing order by repeated maxCoeff (first maximum) and column swaps. */
static void make_jacobi(double x, double y, double z, double* c, double* s) {
    const double deno = 2.0 * fabs(y);
    if (deno < DBL_MIN) {
        *c = 1.0;
        *s = 0.0;
        return;
    }
    const double tau = (x - z) / deno;
    const double w = sqrt(tau * tau + 1.0);
    const double t = tau > 0.0 ? 1.0 / (tau + w) : 1.0 / (tau - w);
    const double sign_t = t > 0.0 ? 1.0 : -1.0;
    const double n = 1.0 / sqrt(t * t + 1.0);
    *s = ((-sign_t * (y / fabs(y))) * fabs(t)) * n;
    *c = n;
}
/* apply_rotation_in_the_plane(x, y, (c, s)): x' = c x + s y, y' = -s x + c y */
static void rot_rows(double m[3][3], int p, int q, double c, double s) {
    for (int j = 0; j < 3; ++j) {
        const double xi = m[p][j], yi = m[q][j];
        m[p][j] = c * xi + s * yi;
        m[q][j] = -s * xi + c * yi;
    }
}
static void rot_cols(double m[3][3], int p, int q, double c, double s) {
    for (int i = 0; i < 3; ++i) {
        const double xi = m[i][p], yi = m[i][q];
        m[i][p] = c * xi + s * yi;
        m[i][q] = -s * xi + c * yi;
    }
}
/* A, U, V row-major 3x3; returns 0, or 1 for a non-finite input (Eigen's InvalidInput) */
int orc_svd3(const double* A, double* U, double* S, double* V) {
    double scale = 0.0;
    for (int i = 0; i < 9; ++i) {
        const double a = fabs(A[i]);
        if (isnan(a)) {
            scale = a;
            break;
        }
        if (a > scale) scale = a;
    }
    if (!isfinite(scale)) return 1;
    if (scale == 0.0) scale = 1.0;
    double w[3][3], u[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}, v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) w[i][j] = A[i * 3 + j] / scale;
    const double precision = 2.0 * DBL_EPSILON, zero = DBL_MIN;
    double max_diag = max_d(max_d(fabs(w[0][0]), fabs(w[1][1])), fabs(w[2][2]));
    int finished = 0;
    for (int sweep = 0; !finished && sweep < JACOBI_MAX_SWEEPS; ++sweep) {
        finished = 1;
        for (int p = 1; p < 3; ++p)
            for (int q = 0; q < p; ++q) {
                const double threshold = max_d(zero, precision * max_diag);
                if (!(fabs(w[p][q]) > threshold || fabs(w[q][p]) > threshold)) continue;
                finished = 0;
                /* real_2x2_jacobi_svd */
                const double m00 = w[p][p], m01 = w[p][q], m10 = w[q][p], m11 = w[q][q];
                const double t = m00 + m11, d = m10 - m01;
                double c1, s1;
                if (fabs(d) < DBL_MIN) {
                    s1 = 0.0;
                    c1 = 1.0;
                } else {
                    const double uu = t / d;
                    const double tmp = sqrt(1.0 + uu * uu);
                    s1 = 1.0 / tmp;
                    c1 = uu / tmp;
                }
                const double n00 = c1 * m00 + s1 * m10, n01 = c1 * m01 + s1 * m11, n11 = -s1 * m01 + c1 * m11;
                double cr, sr;
                make_jacobi(n00, n01, n11, &cr, &sr);
                /* j_left = rot1 * j_right.transpose() */
                const double cl = c1 * cr - s1 * -sr, sl = c1 * -sr + s1 * cr;
                rot_rows(w, p, q, cl, sl);   /* work.applyOnTheLeft(p, q, j_left) */
                rot_cols(u, p, q, cl, sl);   /* U.applyOnTheRight(p, q, j_left.transpose()) */
                rot_cols(w, p, q, cr, -sr);  /* work.applyOnTheRight(p, q, j_right) */
                rot_cols(v, p, q, cr, -sr);  /* V.applyOnTheRight(p, q, j_right) */
                max_diag = max_d(max_diag, max_d(fabs(w[p][p]), fabs(w[q][q])));
            }
    }
    double s[3];
    for (int i = 0; i < 3; ++i) {
        const double a = w[i][i];
        s[i] = fabs(a);
        if (a < 0.0)
            for (int r = 0; r < 3; ++r) u[r][i] = -u[r][i];
    }
    for (int i = 0; i < 3; ++i) s[i] *= scale;
    for (int i = 0; i < 3; ++i) {
        int pos = i;
        for (int j = i + 1; j < 3; ++j)
            if (s[j] > s[pos]) pos = j;
        if (s[pos] == 0.0) break;
        if (pos != i) {
            double tmp = s[i];
            s[i] = s[pos];
            s[pos] = tmp;
            for (int r = 0; r < 3; ++r) {
                tmp = u[r][i];
                u[r][i] = u[r][pos];
                u[r][pos] = tmp;
                tmp = v[r][i];
                v[r][i] = v[r][pos];
                v[r][pos] = tmp;
            }
        }
    }
    for (int i = 0; i < 3; ++i) {
        S[i] = s[i];
        for (int j = 0; j < 3; ++j) {
            U[i * 3 + j] = u[i][j];
            V[i * 3 + j] = v[i][j];
        }
    }
    return 0;
}

/* ---- Eigen 3.4 LDLT<Matrix<double, 6, 6>> (ldlt_inplace<Lower>::unblocked) and _solve_impl ----
 * Returns 0 (Success) or 1 (NumericalIssue: a valid pivot after a zero one, or a zero pivot with a non-zero
 * column below it).  Inner products in index order. */
int orc_ldlt6(const double* A, const double* rhs, double* x) {
    double m[6][6];
    int tr[6];
    int ok = 1, found_zero = 0;
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
            for (int j = 0; j < k; ++j) {
                const double s = m[k][j];
                m[k][j] = m[big][j];
                m[big][j] = s;
            }
            for (int i = big + 1; i < 6; ++i) {
                const double s = m[i][k];
                m[i][k] = m[i][big];
                m[i][big] = s;
            }
            const double s = m[k][k];
            m[k][k] = m[big][big];
            m[big][big] = s;
            for (int i = k + 1; i < big; ++i) {
                const double t = m[i][k];
                m[i][k] = m[big][i];
                m[big][i] = t;
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
        if (valid) {
            for (int i = k + 1; i < 6; ++i) m[i][k] = m[i][k] / akk;
        } else {
            for (int i = k + 1; i < 6; ++i) ok = ok && m[i][k] == 0.0;
        }
        if (found_zero && valid) ok = 0;
        else if (!valid) found_zero = 1;
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
    return ok ? 0 : 1;
}

/* ---- PoseV::exp (transform_vector.cpp:40-60, 96-104); v = (rotation vector, translation) -> row-major 4x4 ---- */
static void skew(const double* v, double a[3][3]) {
    a[0][0] = 0.0, a[0][1] = -v[2], a[0][2] = v[1];
    a[1][0] = v[2], a[1][1] = 0.0, a[1][2] = -v[0];
    a[2][0] = -v[1], a[2][1] = v[0], a[2][2] = 0.0;
}
static void mat3_mul(const double a[3][3], const double b[3][3], double c[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[i][j] = (a[i][0] * b[0][j] + a[i][1] * b[1][j]) + a[i][2] * b[2][j];
}
void orc_posev_exp(const double* v, double* M) {
    const double NUMERIC_EPS = sqrt(DBL_EPSILON), EPS = DBL_EPSILON;
    const double* om = v;
    const double angle = norm3(om);
    const double sa = sin(angle), ca = cos(angle);
    double R[3][3], V[3][3];
    if (angle < NUMERIC_EPS) { /* I + skew(v) */
        double s[3][3];
        skew(om, s);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i][j] = (i == j ? 1.0 : 0.0) + s[i][j];
    } else { /* I + sin A + ((1 - cos) A) A, A = skew(v / angle) */
        const double ax[3] = {om[0] / angle, om[1] / angle, om[2] / angle};
        double a[3][3], b[3][3], bb[3][3];
        skew(ax, a);
        const double c1 = 1.0 - ca;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) b[i][j] = c1 * a[i][j];
        mat3_mul(b, a, bb);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i][j] = ((i == j ? 1.0 : 0.0) + sa * a[i][j]) + bb[i][j];
    }
    if (angle < EPS) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) V[i][j] = i == j ? 1.0 : 0.0;
    } else { /* I + ((1 - cos) A) / angle + (((angle - sin) A) A) / angle */
        const double ax[3] = {om[0] / angle, om[1] / angle, om[2] / angle};
        double a[3][3], b[3][3], bb[3][3];
        skew(ax, a);
        const double c1 = 1.0 - ca, c2 = angle - sa;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) b[i][j] = c2 * a[i][j];
        mat3_mul(b, a, bb);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) V[i][j] = ((i == j ? 1.0 : 0.0) + (c1 * a[i][j]) / angle) + bb[i][j] / angle;
    }
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) M[i * 4 + j] = R[i][j];
        M[i * 4 + 3] = (V[i][0] * v[3] + V[i][1] * v[4]) + V[i][2] * v[5];
    }
    M[12] = M[13] = M[14] = 0.0;
    M[15] = 1.0;
}

/* a = b * a for row-major 4x4 (PoseH(delta) * current_pose) */
static void pose_premul(const double* b, double* a) {
    double r[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            r[i * 4 + j] = ((b[i * 4] * a[j] + b[i * 4 + 1] * a[4 + j]) + b[i * 4 + 2] * a[8 + j]) + b[i * 4 + 3] * a[12 + j];
    memcpy(a, r, sizeof(r));
}
/* x = R p + t for the top 3x4 of a row-major pose */
static void transform(const double* pose, const double* p, double* x) {
    for (int d = 0; d < 3; ++d)
        x[d] = ((pose[d * 4] * p[0] + pose[d * 4 + 1] * p[1]) + pose[d * 4 + 2] * p[2]) + pose[d * 4 + 3];
}
static void rotate(const double* pose, const double* p, double* x) {
    for (int d = 0; d < 3; ++d) x[d] = (pose[d * 4] * p[0] + pose[d * 4 + 1] * p[1]) + pose[d * 4 + 2] * p[2];
}

/* MAD-scaled Huber threshold (:1650-1655, :1823-1828) */
static double huber_delta(const double* r, size_t k, double max_corr_dist) {
    const double mad = orc_median_abs(r, k);
    double sigma = MAD_TO_SIGMA * mad;
    if (!isfinite(sigma) || sigma < 1e-4) sigma = max_d(1e-3, 0.25 * max_corr_dist);
    return HUBER_K * sigma;
}
static double huber_w(double r, double delta) {
    const double abs_r = fabs(r);
    return (abs_r <= delta || delta <= 0.0) ? 1.0 : (delta / abs_r);
}

/* point_to_point_align (:1590-1722).  Returns 0, or -1 for "max_corr_dist must be finite and greater than zero".
 * *iterations = the iterations that reached the solve (the SVD). */
int orc_point_to_point_align(const double* src, size_t n, const double* tgt, size_t m, const double* guess,
                             double max_corr_dist, double* out, int* iterations) {
    if (!isfinite(max_corr_dist) || max_corr_dist <= 0.0) return -1;
    memcpy(out, guess, 16 * sizeof(double));
    *iterations = 0;
    if (n < MIN_ICP_POINTS || m < MIN_ICP_POINTS) return 0;
    double pose[16];
    memcpy(pose, guess, sizeof(pose));
    int solved_any_level = 0;
    const double corr_dist_sq = max_corr_dist * max_corr_dist;
    Grid g;
    grid_build(&g, tgt, NULL, m, max_corr_dist);
    double *cx = malloc(n * 3 * sizeof(double)), *cq = malloc(n * 3 * sizeof(double)), *cr = malloc(n * sizeof(double));
    double* cw = malloc(n * sizeof(double));
    for (int iter = 0; iter < ICP_MAX_ITERATIONS; ++iter) {
        size_t k = 0;
        for (size_t i = 0; i < n; ++i) {
            double x[3];
            transform(pose, src + 3 * i, x);
            const int nn = grid_nearest(&g, tgt, x, corr_dist_sq);
            if (nn < 0) continue;
            const double* q = tgt + 3 * (size_t)nn;
            const double d[3] = {x[0] - q[0], x[1] - q[1], x[2] - q[2]};
            const double r = norm3(d);
            if (!finite3(x) || !finite3(q) || !isfinite(r)) continue;
            memcpy(cx + 3 * k, x, sizeof(x));
            memcpy(cq + 3 * k, q, 3 * sizeof(double));
            cr[k++] = r;
        }
        if (k < MIN_ICP_POINTS) break;
        solved_any_level = 1;
        const double delta = huber_delta(cr, k, max_corr_dist);
        double wsum = 0.0, mx[3] = {0, 0, 0}, mq[3] = {0, 0, 0};
        for (size_t i = 0; i < k; ++i) {
            const double w = huber_w(cr[i], delta);
            cw[i] = w;
            wsum += w;
            for (int d = 0; d < 3; ++d) {
                mx[d] += w * cx[3 * i + d];
                mq[d] += w * cq[3 * i + d];
            }
        }
        if (!isfinite(wsum) || wsum <= 1e-12) break;
        for (int d = 0; d < 3; ++d) {
            mx[d] /= wsum;
            mq[d] /= wsum;
        }
        double cov[9] = {0};
        for (size_t i = 0; i < k; ++i) {
            double a[3], b[3];
            for (int d = 0; d < 3; ++d) {
                a[d] = cw[i] * (cx[3 * i + d] - mx[d]);
                b[d] = cq[3 * i + d] - mq[d];
            }
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) cov[r * 3 + c] += a[r] * b[c];
        }
        ++*iterations;
        double U[9], S[3], V[9];
        const int bad = orc_svd3(cov, U, S, V);
        int finite_uv = !bad;
        for (int i = 0; i < 9 && finite_uv; ++i) finite_uv = isfinite(U[i]) && isfinite(V[i]);
        if (!finite_uv) break;
        double R[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i * 3 + j] = (V[i * 3] * U[j * 3] + V[i * 3 + 1] * U[j * 3 + 1]) + V[i * 3 + 2] * U[j * 3 + 2];
        /* Eigen's 3x3 determinant (bruteforce_det3_helper) */
        const double det = (R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6])) +
                           R[2] * (R[3] * R[7] - R[4] * R[6]);
        if (det < 0.0) {
            for (int i = 0; i < 3; ++i) V[i * 3 + 2] *= -1.0;
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j)
                    R[i * 3 + j] = (V[i * 3] * U[j * 3] + V[i * 3 + 1] * U[j * 3 + 1]) + V[i * 3 + 2] * U[j * 3 + 2];
        }
        double dt[3];
        for (int d = 0; d < 3; ++d) dt[d] = mq[d] - ((R[d * 3] * mx[0] + R[d * 3 + 1] * mx[1]) + R[d * 3 + 2] * mx[2]);
        int finite_r = 1;
        for (int i = 0; i < 9; ++i) finite_r = finite_r && isfinite(R[i]);
        if (!finite_r || !finite3(dt)) break;
        const double D[16] = {R[0], R[1], R[2], dt[0], R[3], R[4], R[5], dt[1], R[6], R[7], R[8], dt[2], 0, 0, 0, 1};
        pose_premul(D, pose);
        const double trace_term = max_d(-1.0, min_d(0.5 * ((R[0] + R[4]) + R[8] - 1.0), 1.0));
        if (acos(trace_term) < 1e-4 && norm3(dt) < 1e-3) break;
    }
    free(cx);
    free(cq);
    free(cr);
    free(cw);
    grid_free(&g);
    if (solved_any_level) memcpy(out, pose, sizeof(pose));
    return 0;
}

/* point_to_plane_align (:1724-1874).  Returns 0, or the first failed check: -1 "max_corr_dist must be finite and
 * greater than zero", -2 "max_normal_angle_deg must be finite and in [0, 180]", -3 source rows, -4 target rows. */
int orc_point_to_plane_align(const double* src, size_t n, const double* tgt, size_t m, const double* sn, size_t n_sn,
                             const double* tn, size_t n_tn, const double* guess, double max_corr_dist,
                             double max_normal_angle_deg, double* out, int* iterations) {
    if (!isfinite(max_corr_dist) || max_corr_dist <= 0.0) return -1;
    if (!isfinite(max_normal_angle_deg) || max_normal_angle_deg < 0.0 || max_normal_angle_deg > 180.0) return -2;
    if (n != n_sn) return -3;
    if (m != n_tn) return -4;
    memcpy(out, guess, 16 * sizeof(double));
    *iterations = 0;
    if (n < MIN_ICP_POINTS || m < MIN_ICP_POINTS) return 0;
    double pose[16];
    memcpy(pose, guess, sizeof(pose));
    int solved_any_level = 0;
    const double corr_dist_sq = max_corr_dist * max_corr_dist;
    const double cos_angle_gate = cos(max_normal_angle_deg * 3.14159265358979323846 / 180.0);
    Grid g;
    grid_build(&g, tgt, tn, m, max_corr_dist);
    double *cx = malloc(n * 3 * sizeof(double)), *cn = malloc(n * 3 * sizeof(double)), *cr = malloc(n * sizeof(double));
    for (int iter = 0; iter < ICP_MAX_ITERATIONS; ++iter) {
        size_t k = 0;
        for (size_t i = 0; i < n; ++i) {
            double ns[3] = {sn[3 * i], sn[3 * i + 1], sn[3 * i + 2]};
            const double ns_norm = norm3(ns);
            if (!finite3(ns) || ns_norm <= NORMAL_EPS) continue;
            for (int d = 0; d < 3; ++d) ns[d] /= ns_norm;
            double x[3], nw[3];
            transform(pose, src + 3 * i, x);
            rotate(pose, ns, nw);
            const int nn = grid_nearest(&g, tgt, x, corr_dist_sq);
            if (nn < 0) continue;
            const double* q = tgt + 3 * (size_t)nn;
            double nt[3] = {tn[3 * (size_t)nn], tn[3 * (size_t)nn + 1], tn[3 * (size_t)nn + 2]};
            const double nt_norm = norm3(nt);
            if (!finite3(nt) || nt_norm <= NORMAL_EPS) continue;
            for (int d = 0; d < 3; ++d) nt[d] /= nt_norm;
            const double n_align = fabs(dot3(nt, nw));
            if (!isfinite(n_align) || n_align < cos_angle_gate) continue;
            const double d[3] = {x[0] - q[0], x[1] - q[1], x[2] - q[2]};
            const double r = dot3(nt, d);
            if (!isfinite(r)) continue;
            memcpy(cx + 3 * k, x, sizeof(x));
            memcpy(cn + 3 * k, nt, sizeof(nt));
            cr[k++] = r;
        }
        if (k < MIN_ICP_POINTS) break;
        solved_any_level = 1;
        const double delta = huber_delta(cr, k, max_corr_dist);
        double H[36] = {0}, b[6] = {0};
        for (size_t i = 0; i < k; ++i) {
            const double w = huber_w(cr[i], delta);
            const double* x = cx + 3 * i;
            const double* nv = cn + 3 * i;
            const double J[6] = {x[1] * nv[2] - x[2] * nv[1], x[2] * nv[0] - x[0] * nv[2], x[0] * nv[1] - x[1] * nv[0],
                                 nv[0], nv[1], nv[2]};
            for (int r = 0; r < 6; ++r) {
                for (int c = 0; c < 6; ++c) H[r * 6 + c] += w * (J[r] * J[c]);
                b[r] += -w * (J[r] * cr[i]);
            }
        }
        for (int d = 0; d < 6; ++d) H[d * 6 + d] += 1e-10;
        ++*iterations;
        double dx[6];
        if (orc_ldlt6(H, b, dx) != 0) break;
        int finite_dx = 1;
        for (int d = 0; d < 6; ++d) finite_dx = finite_dx && isfinite(dx[d]);
        if (!finite_dx) break;
        double E[16];
        orc_posev_exp(dx, E);
        pose_premul(E, pose);
        if (norm3(dx) < 1e-4 && norm3(dx + 3) < 1e-3) break;
    }
    free(cx);
    free(cn);
    free(cr);
    grid_free(&g);
    if (solved_any_level) memcpy(out, pose, sizeof(pose));
    return 0;
}
