/* orc_ground.c -- CPU oracle of ground segmentation (test infrastructure only).
 *
 * Restates ouster_algorithm/src/ground_seg.cpp:179-1314 (build_lower_envelope_ground_model, the grid passes,
 * xy_point_is_ground_like and get_ground_mask_into) in plain C, double precision, one rounding per operation
 * (built with -ffp-contract=off).  Inputs are one frame's range images, status, LUT, column poses and, optionally,
 * normals for the first two returns; the caller computes normals when it wants them (oracle/ground.py).
 *
 * Orders the reference leaves unspecified are pinned (DESIGN §9):
 *  - every selection (nth_element) is taken on values sorted in the total order "<, then -0.0 before +0.0", so
 *    the selected bits are defined when a set holds both zeros;
 *  - the x / y extents are the minimum and maximum in that order too;
 *  - the fallback ground z sums zs[low..high] in ascending order;
 *  - components are numbered by their lowest cell index; the main one is the first of the largest.
 *
 * orc_ground_run() can stop after any grid pass (ORC_GROUND_STAGE_*) and returns the model at that point, so tests
 * can compare the GPU pass by pass.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum {
    STAGE_CELLS = 0, STAGE_FILL1, STAGE_SMOOTH1, STAGE_PRUNE, STAGE_FILL2, STAGE_SMOOTH2, STAGE_COMPONENTS,
    STAGE_FILL3
};

typedef struct orc_ground_frame {
    int h, w, n_returns;
    int pad;
    const uint32_t* const* range; /* n_returns images, h x w */
    const uint32_t* status;       /* w */
    const double* dir;            /* h*w x 3 */
    const double* off;            /* h*w x 3 */
    const double* poses;          /* w x 16, row-major */
    const double* normals[2];     /* h*w x 3 for returns 0 and 1, or NULL */
    double grid_size;
} orc_ground_frame;

typedef struct orc_ground_model {
    double origin_x, origin_y, fallback_z, footprint_bound;
    int32_t rows, cols, valid, has_columns;
} orc_ground_model;

#define NAN_D ((double)NAN)

/* ---- constants of ground_seg.cpp:43-156 ---- */
static const double MIN_RANGE_M = 0.15, NORMAL_EPS = 1e-6, MAD_TO_SIGMA = 1.4826;
static const double XY_BOUNDS_PERCENTILE = 0.95, INDOOR_BOUND_M = 25.0, INDOOR_MAX_Z = 0.3;
static const double TAIL_LOW = 0.01, TAIL_HIGH = 0.20;
static const double CELL_LOW_PCT = 0.15, ROUGH_BAND_M = 0.45;
static const double NZ_PREFILTER = 0.15, POINT_NZ_MIN = 0.15, WALL_NZ_MAX = 0.45, WALL_ABOVE_LOCAL = 0.20;
static const size_t NF_MIN_POINTS = 4;
static const double FILL_MAX_SPREAD = 0.65, SMOOTH_MAX_DIFF = 0.55;
static const double ANCHOR_ABOVE = 1.10, MAX_NEIGHBOR_STEP = 0.75, SLOPE_PER_M = 0.80, PRUNE_MIN_ABOVE = 1.50;
static const double COMP_CLOSE = 0.50, COMP_HIGH = 1.20, COMP_MODERATE_FRAC = 0.20, COMP_HIGH_FRAC = 0.80,
                    COMP_MAX_STEP = 0.45;
static const int LOOKUP_RADIUS = 8;
static const double BASE_TOL = 0.50, ROUGH_K = 2.5, NOISE_K = 0.01, NOISE_MAX = 0.50, LOOKUP_TOL_PER_M = 0.20,
                    LOOKUP_TOL_MAX = 0.45, OUTDOOR_MAX_Z = 1.20, MAX_ABOVE_LOCAL = 0.50, MAX_BELOW_LOCAL = 1.20,
                    UNSUPPORTED_ABOVE = 0.90;
static const double FLOOR_PCT = 0.05, OBST_SPAN = 0.55, OBST_MIN_ABOVE = 0.25, OBST_ROUGH_CAP = 0.10,
                    OBST_WALL_NZ = 0.65, OBST_WALL_ABOVE = 0.20, LIFT_MAX = 0.25, WALL_FLOOR_HARD = 0.35;
static const size_t OBST_MIN_POINTS = 2;
static const int DR[8] = {-1, -1, -1, 0, 0, 1, 1, 1}, DC[8] = {-1, 0, 1, -1, 1, -1, 0, 1};

/* ---- selections ---- */
static int cmp_total(const void* pa, const void* pb) {
    const double a = *(const double*)pa, b = *(const double*)pb;
    if (a < b) return -1;
    if (a > b) return 1;
    return (int)(signbit(b) != 0) - (int)(signbit(a) != 0);
}
static void sort_d(double* v, size_t n) { qsort(v, n, sizeof(double), cmp_total); }
static double kth(double* v, size_t n, size_t k) {
    sort_d(v, n);
    return v[k];
}
static double median_value(double* v, size_t n) { return n == 0 ? NAN_D : kth(v, n, n / 2u); }
static double robust_spread(double* v, size_t n, double center) {
    if (n < 2u || !isfinite(center)) return 0.0;
    for (size_t i = 0; i < n; ++i) v[i] = fabs(v[i] - center);
    const double mad = median_value(v, n);
    return isfinite(mad) ? MAD_TO_SIGMA * mad : 0.0;
}
static double percentile_value(double* v, size_t n, double pct) {
    if (n == 0) return NAN_D;
    pct = fmin(1.0, fmax(0.0, pct));
    size_t idx = (size_t)floor(pct * (double)(n - 1));
    if (idx > n - 1) idx = n - 1;
    return kth(v, n, idx);
}
static int finite3(const double* p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }
static double norm3(const double* p) { return sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]); }

static double abs_normal_z(const double* n) {
    if (n == NULL || !finite3(n)) return NAN_D;
    const double nn = norm3(n);
    if (nn <= NORMAL_EPS) return NAN_D;
    return fabs(n[2] / nn);
}

/* ---- model ---- */
typedef struct Model {
    orc_ground_model m;
    double cell, inv;
    int indoor;
    uint8_t *valid, *obstacle;
    double *floor_z, *height, *rough;
} Model;

#define IDX(r, c) ((size_t)(r) * (size_t)cols + (size_t)(c))

static void fill_holes(Model* M, int radius) {
    if (!M->m.valid) return;
    const int rows = M->m.rows, cols = M->m.cols;
    const size_t n = (size_t)rows * cols;
    uint8_t* fv = malloc(n);
    double* fh = malloc(n * sizeof(double));
    double* fr = malloc(n * sizeof(double));
    memcpy(fv, M->valid, n);
    memcpy(fh, M->height, n * sizeof(double));
    memcpy(fr, M->rough, n * sizeof(double));
    const size_t cap = (size_t)(2 * radius + 1) * (2 * radius + 1);
    double* hs = malloc(cap * sizeof(double));
    double* hc = malloc(cap * sizeof(double));
    double* rs = malloc(cap * sizeof(double));
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) {
            const size_t idx = IDX(r, c);
            if (M->valid[idx]) continue;
            size_t k = 0;
            for (int dr = -radius; dr <= radius; ++dr)
                for (int dc = -radius; dc <= radius; ++dc) {
                    if (dr == 0 && dc == 0) continue;
                    const int rr = r + dr, cc = c + dc;
                    if (rr < 0 || rr >= rows || cc < 0 || cc >= cols) continue;
                    const size_t ni = IDX(rr, cc);
                    if (!M->valid[ni] || !isfinite(M->height[ni])) continue;
                    hs[k] = M->height[ni];
                    rs[k] = M->rough[ni];
                    ++k;
                }
            if (k == 0) continue;
            memcpy(hc, hs, k * sizeof(double));
            const double fill_h = median_value(hc, k);
            const double spread = robust_spread(hs, k, fill_h);
            if (!isfinite(fill_h) || spread > FILL_MAX_SPREAD) continue;
            fh[idx] = fill_h;
            fr[idx] = median_value(rs, k);
            fv[idx] = 1;
        }
    memcpy(M->valid, fv, n);
    memcpy(M->height, fh, n * sizeof(double));
    memcpy(M->rough, fr, n * sizeof(double));
    free(fv), free(fh), free(fr), free(hs), free(hc), free(rs);
}

static void smooth(Model* M) {
    if (!M->m.valid) return;
    const int rows = M->m.rows, cols = M->m.cols;
    const size_t n = (size_t)rows * cols;
    double* sh = malloc(n * sizeof(double));
    double* sr = malloc(n * sizeof(double));
    memcpy(sh, M->height, n * sizeof(double));
    memcpy(sr, M->rough, n * sizeof(double));
    double hs[9], rs[9];
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) {
            const size_t idx = IDX(r, c);
            if (!M->valid[idx] || !isfinite(M->height[idx])) continue;
            const double ch = M->height[idx];
            size_t k = 0;
            for (int dr = -1; dr <= 1; ++dr)
                for (int dc = -1; dc <= 1; ++dc) {
                    const int rr = r + dr, cc = c + dc;
                    if (rr < 0 || rr >= rows || cc < 0 || cc >= cols) continue;
                    const size_t ni = IDX(rr, cc);
                    if (!M->valid[ni] || !isfinite(M->height[ni])) continue;
                    if (fabs(M->height[ni] - ch) > SMOOTH_MAX_DIFF) continue;
                    hs[k] = M->height[ni];
                    rs[k] = M->rough[ni];
                    ++k;
                }
            if (k) {
                sh[idx] = median_value(hs, k);
                sr[idx] = median_value(rs, k);
            }
        }
    memcpy(M->height, sh, n * sizeof(double));
    memcpy(M->rough, sr, n * sizeof(double));
    free(sh), free(sr);
}

static void invalidate(Model* M, size_t idx) {
    M->valid[idx] = 0;
    M->height[idx] = NAN_D;
    M->rough[idx] = 0.0;
}

static void prune(Model* M) {
    if (!M->m.valid || !isfinite(M->m.fallback_z)) return;
    const int rows = M->m.rows, cols = M->m.cols;
    const size_t n = (size_t)rows * cols;
    uint8_t* reach = calloc(n, 1);
    size_t* queue = malloc(n * sizeof(size_t));
    size_t qn = 0;
    for (size_t i = 0; i < n; ++i) {
        if (!M->valid[i] || !isfinite(M->height[i])) continue;
        if (M->height[i] <= M->m.fallback_z + ANCHOR_ABOVE) {
            reach[i] = 1;
            queue[qn++] = i;
        }
    }
    if (qn > 0) {
        double dist[8];
        for (int d = 0; d < 8; ++d) dist[d] = M->cell * sqrt((double)(DR[d] * DR[d] + DC[d] * DC[d]));
        for (size_t head = 0; head < qn; ++head) {
            const size_t idx = queue[head];
            const int r = (int)(idx / (size_t)cols), c = (int)(idx % (size_t)cols);
            const double h = M->height[idx];
            for (int d = 0; d < 8; ++d) {
                const int rr = r + DR[d], cc = c + DC[d];
                if (rr < 0 || rr >= rows || cc < 0 || cc >= cols) continue;
                const size_t ni = IDX(rr, cc);
                if (reach[ni] || !M->valid[ni] || !isfinite(M->height[ni])) continue;
                const double allowed = fmin(MAX_NEIGHBOR_STEP, 0.25 + SLOPE_PER_M * dist[d]);
                if (fabs(M->height[ni] - h) > allowed) continue;
                if (M->height[ni] - h > 0.50 && M->obstacle[ni]) continue;
                reach[ni] = 1;
                queue[qn++] = ni;
            }
        }
        for (size_t i = 0; i < n; ++i) {
            if (!M->valid[i] || !isfinite(M->height[i])) continue;
            if (!reach[i] && M->height[i] > M->m.fallback_z + PRUNE_MIN_ABOVE) invalidate(M, i);
        }
    }
    free(reach), free(queue);
}

static void reject_components(Model* M) {
    if (!M->m.valid || !isfinite(M->m.fallback_z)) return;
    const int rows = M->m.rows, cols = M->m.cols;
    const size_t n = (size_t)rows * cols;
    int* label = malloc(n * sizeof(int));
    size_t* order = malloc(n * sizeof(size_t)); /* cells grouped by component, components in label order */
    size_t* start = malloc((n + 1) * sizeof(size_t));
    double* hs = malloc(n * sizeof(double));
    for (size_t i = 0; i < n; ++i) label[i] = -1;
    size_t nc = 0, qn = 0;
    for (size_t s = 0; s < n; ++s) {
        if (!M->valid[s] || !isfinite(M->height[s]) || label[s] >= 0) continue;
        start[nc] = qn;
        label[s] = (int)nc;
        order[qn++] = s;
        for (size_t head = start[nc]; head < qn; ++head) {
            const size_t idx = order[head];
            const int r = (int)(idx / (size_t)cols), c = (int)(idx % (size_t)cols);
            for (int d = 0; d < 8; ++d) {
                const int rr = r + DR[d], cc = c + DC[d];
                if (rr < 0 || rr >= rows || cc < 0 || cc >= cols) continue;
                const size_t ni = IDX(rr, cc);
                if (label[ni] >= 0 || !M->valid[ni] || !isfinite(M->height[ni])) continue;
                if (fabs(M->height[ni] - M->height[idx]) > COMP_MAX_STEP) continue;
                label[ni] = (int)nc;
                order[qn++] = ni;
            }
        }
        ++nc;
    }
    start[nc] = qn;
    double* med = malloc((nc + 1) * sizeof(double));
    long main_id = -1;
    size_t main_size = 0;
    double main_med = M->m.fallback_z;
    for (size_t ci = 0; ci < nc; ++ci) {
        const size_t k = start[ci + 1] - start[ci];
        for (size_t j = 0; j < k; ++j) hs[j] = M->height[order[start[ci] + j]];
        med[ci] = median_value(hs, k);
        if (!isfinite(med[ci])) continue;
        if (med[ci] <= M->m.fallback_z + ANCHOR_ABOVE && k > main_size) {
            main_id = (long)ci;
            main_size = k;
            main_med = med[ci];
        }
    }
    if (main_id >= 0) {
        for (size_t ci = 0; ci < nc; ++ci) {
            if ((long)ci == main_id || !isfinite(med[ci])) continue;
            const size_t k = start[ci + 1] - start[ci];
            const double dz = med[ci] - main_med;
            const double frac = (double)k / (double)main_size;
            if (fabs(dz) <= COMP_CLOSE) continue;
            if (dz > COMP_CLOSE && dz <= COMP_HIGH && frac >= COMP_MODERATE_FRAC) continue;
            if (dz > COMP_HIGH && frac >= COMP_HIGH_FRAC) continue;
            if (dz < -COMP_CLOSE && dz >= -COMP_HIGH) continue;
            for (size_t j = start[ci]; j < start[ci + 1]; ++j) invalidate(M, order[j]);
        }
    }
    free(label), free(order), free(start), free(hs), free(med);
}

/* one point of one return: dewarped XYZ (cartesianT then dewarp, ob_project.cuh rounding) */
static void point_of(const orc_ground_frame* f, const uint32_t* range, int row, int col, double* p) {
    const size_t i = (size_t)row * f->w + col;
    const uint32_t r = range[i];
    double q[3];
    for (int k = 0; k < 3; ++k) q[k] = r == 0 ? 0.0 : (double)r * f->dir[i * 3 + k] + f->off[i * 3 + k];
    const double* m = f->poses + (size_t)col * 16;
    for (int k = 0; k < 3; ++k) {
        const double a = m[k * 4] * q[0], b = m[k * 4 + 1] * q[1], c = m[k * 4 + 2] * q[2];
        p[k] = (a + (b + c)) + m[k * 4 + 3];
    }
}

typedef struct Vec {
    double* v;
    size_t n, cap;
} Vec;
static void push(Vec* a, double x) {
    if (a->n == a->cap) {
        a->cap = a->cap ? a->cap * 2 : 8;
        a->v = realloc(a->v, a->cap * sizeof(double));
    }
    a->v[a->n++] = x;
}

static int model_point_ok(const orc_ground_frame* f, int ret, int row, int col, int first, int last, double* p) {
    if (col < first || col > last || f->status[col] == 0u) return 0;
    if (f->range[ret][(size_t)row * f->w + col] == 0u) return 0;
    point_of(f, f->range[ret], row, col, p);
    return finite3(p) && !(norm3(p) < MIN_RANGE_M);
}

/* build_lower_envelope_ground_model (ground_seg.cpp:666-945), stopping after pass `stop` */
static void build_model(const orc_ground_frame* f, int first, int last, int stop, Model* M) {
    const int H = f->h, W = f->w;
    const int n_model = f->n_returns >= 2 ? 2 : 1;
    double min_x = INFINITY, min_y = INFINITY, max_x = -INFINITY, max_y = -INFINITY;
    Vec zs = {0}, fp = {0};
    double p[3];
    for (int ret = 0; ret < n_model; ++ret)
        for (int col = first; col <= last; ++col)
            for (int row = 0; row < H; ++row) {
                if (!model_point_ok(f, ret, row, col, first, last, p)) continue;
                min_x = cmp_total(&p[0], &min_x) < 0 ? p[0] : min_x;
                min_y = cmp_total(&p[1], &min_y) < 0 ? p[1] : min_y;
                max_x = cmp_total(&p[0], &max_x) > 0 ? p[0] : max_x;
                max_y = cmp_total(&p[1], &max_y) > 0 ? p[1] : max_y;
                push(&zs, p[2]);
                push(&fp, fmax(fabs(p[0]), fabs(p[1])));
            }
    if (zs.n == 0) {
        free(zs.v), free(fp.v);
        return;
    }
    {
        size_t k = (size_t)floor(XY_BOUNDS_PERCENTILE * (double)(fp.n - 1));
        if (k > fp.n - 1) k = fp.n - 1;
        M->m.footprint_bound = kth(fp.v, fp.n, k);
    }
    {
        const size_t n = zs.n;
        size_t lo = (size_t)floor(TAIL_LOW * (double)(n - 1)), hi = (size_t)ceil(TAIL_HIGH * (double)(n - 1));
        if (lo > n - 1) lo = n - 1;
        if (hi > n - 1) hi = n - 1;
        if (hi < lo) hi = lo;
        sort_d(zs.v, n);
        double sum = 0.0;
        for (size_t i = lo; i <= hi; ++i) sum += zs.v[i];
        M->m.fallback_z = sum / (double)(hi - lo + 1);
    }
    M->cell = f->grid_size;
    M->inv = 1.0 / f->grid_size;
    M->m.origin_x = floor(min_x * M->inv) * M->cell;
    M->m.origin_y = floor(min_y * M->inv) * M->cell;
    int cols = (int)ceil((max_x - M->m.origin_x) / M->cell) + 1;
    int rows = (int)ceil((max_y - M->m.origin_y) / M->cell) + 1;
    M->m.cols = cols = cols > 1 ? cols : 1;
    M->m.rows = rows = rows > 1 ? rows : 1;
    const size_t n = (size_t)rows * cols;
    M->valid = calloc(n, 1);
    M->obstacle = calloc(n, 1);
    M->floor_z = malloc(n * sizeof(double));
    M->height = malloc(n * sizeof(double));
    M->rough = calloc(n, sizeof(double));
    for (size_t i = 0; i < n; ++i) M->floor_z[i] = M->height[i] = NAN_D;
    Vec* cz = calloc(n, sizeof(Vec));
    Vec* nz = calloc(n, sizeof(Vec));
    for (int ret = 0; ret < n_model; ++ret) {
        const double* nrm = f->normals[ret];
        for (int col = first; col <= last; ++col)
            for (int row = 0; row < H; ++row) {
                if (!model_point_ok(f, ret, row, col, first, last, p)) continue;
                const int cc = (int)floor((p[0] - M->m.origin_x) * M->inv);
                const int rr = (int)floor((p[1] - M->m.origin_y) * M->inv);
                if (rr < 0 || rr >= rows || cc < 0 || cc >= cols) continue;
                const size_t ci = IDX(rr, cc);
                push(&cz[ci], p[2]);
                if (nrm != NULL) {
                    const double* nv = nrm + ((size_t)row * W + col) * 3;
                    const double nn = norm3(nv);
                    if (finite3(nv) && nn > NORMAL_EPS && fabs(nv[2] / nn) >= NZ_PREFILTER) push(&nz[ci], p[2]);
                }
            }
    }
    const int any_normals = f->normals[0] != NULL || f->normals[1] != NULL;
    size_t valid_cells = 0;
    Vec work = {0};
    for (size_t ci = 0; ci < n; ++ci) {
        Vec* z = &cz[ci];
        if (z->n == 0) continue;
        work.n = 0;
        for (size_t j = 0; j < z->n; ++j) push(&work, z->v[j]);
        sort_d(work.v, work.n);
        const size_t m = work.n;
        const double z_max = work.v[m - 1];
        size_t fi = (size_t)floor(FLOOR_PCT * (double)(m - 1)), hi = (size_t)floor(CELL_LOW_PCT * (double)(m - 1));
        if (fi > m - 1) fi = m - 1;
        if (hi > m - 1) hi = m - 1;
        const double floor_z = work.v[fi], h_all = work.v[hi];
        if (!isfinite(h_all) || !isfinite(floor_z)) continue;
        M->floor_z[ci] = floor_z;
        size_t above = 0;
        for (size_t j = 0; j < m; ++j)
            if (isfinite(z->v[j]) && z->v[j] > floor_z + OBST_MIN_ABOVE) ++above;
        const int obstacle = (z_max - floor_z) > OBST_SPAN && above >= OBST_MIN_POINTS;
        if (obstacle) M->obstacle[ci] = 1;
        double h_f = NAN_D;
        int use_f = 0;
        if (any_normals && nz[ci].n >= NF_MIN_POINTS) {
            double* tmp = malloc(nz[ci].n * sizeof(double));
            memcpy(tmp, nz[ci].v, nz[ci].n * sizeof(double));
            h_f = percentile_value(tmp, nz[ci].n, CELL_LOW_PCT);
            free(tmp);
            const int lifted = isfinite(h_f) && h_f > h_all + LIFT_MAX;
            use_f = isfinite(h_f) && !lifted && !obstacle;
        }
        const Vec* sel = use_f ? &nz[ci] : z;
        const double h = obstacle ? floor_z : (use_f ? h_f : h_all);
        if (!isfinite(h) || sel->n == 0) continue;
        double* band = malloc(sel->n * sizeof(double));
        size_t nb = 0;
        for (size_t j = 0; j < sel->n; ++j)
            if (isfinite(sel->v[j]) && sel->v[j] <= h + ROUGH_BAND_M) band[nb++] = sel->v[j];
        if (nb == 0) band[nb++] = h;
        double rough = robust_spread(band, nb, h);
        free(band);
        if (obstacle) rough = fmin(rough, OBST_ROUGH_CAP);
        M->valid[ci] = 1;
        M->height[ci] = h;
        M->rough[ci] = rough;
        ++valid_cells;
    }
    for (size_t ci = 0; ci < n; ++ci) free(cz[ci].v), free(nz[ci].v);
    free(cz), free(nz), free(work.v), free(zs.v), free(fp.v);
    if (valid_cells == 0) return;
    M->m.valid = 1;
    if (stop >= STAGE_FILL1) fill_holes(M, 6);
    if (stop >= STAGE_SMOOTH1) smooth(M);
    if (stop >= STAGE_PRUNE) prune(M);
    if (stop >= STAGE_FILL2) fill_holes(M, 6);
    if (stop >= STAGE_SMOOTH2) smooth(M);
    if (stop >= STAGE_COMPONENTS) reject_components(M);
    if (stop >= STAGE_FILL3) fill_holes(M, 3);
}

/* xy_point_is_ground_like (ground_seg.cpp:947-1088) */
static int ground_like(const Model* M, const double* p, double range, double fallback, const double* nrm) {
    const int rows = M->m.rows, cols = M->m.cols;
    const double eff = isfinite(M->m.fallback_z) ? M->m.fallback_z : fallback;
    if (M->indoor && isfinite(eff) && p[2] > eff + INDOOR_MAX_Z) return 0;
    int in_grid = 0, cr = 0, cc = 0;
    if (M->m.valid && finite3(p)) {
        cc = (int)floor((p[0] - M->m.origin_x) * M->inv);
        cr = (int)floor((p[1] - M->m.origin_y) * M->inv);
        in_grid = cr >= 0 && cr < rows && cc >= 0 && cc < cols;
    }
    if (in_grid) {
        const size_t ci = IDX(cr, cc);
        if (M->obstacle[ci] && isfinite(M->floor_z[ci])) {
            const double above = p[2] - M->floor_z[ci];
            if (above > WALL_FLOOR_HARD) return 0;
            const double nz = abs_normal_z(nrm);
            if (isfinite(nz) && nz < OBST_WALL_NZ && above > OBST_WALL_ABOVE) return 0;
        }
        double lh = NAN_D, lr = 0.0, ld = 0.0;
        int found = 0;
        if (M->valid[ci] && isfinite(M->height[ci])) {
            lh = M->height[ci];
            lr = M->rough[ci];
            found = 1;
        } else {
            double best = INFINITY;
            size_t bi = 0;
            for (int rad = 1; rad <= LOOKUP_RADIUS && !found; ++rad) {
                for (int dr = -rad; dr <= rad; ++dr)
                    for (int dc = -rad; dc <= rad; ++dc) {
                        if ((abs(dr) > abs(dc) ? abs(dr) : abs(dc)) != rad) continue;
                        const int rr = cr + dr, c2 = cc + dc;
                        if (rr < 0 || rr >= rows || c2 < 0 || c2 >= cols) continue;
                        const size_t ni = IDX(rr, c2);
                        if (!M->valid[ni] || !isfinite(M->height[ni])) continue;
                        const double d2 = (double)(dr * dr + dc * dc);
                        if (d2 < best) {
                            best = d2;
                            bi = ni;
                            found = 1;
                        }
                    }
                if (found) {
                    lh = M->height[bi];
                    lr = M->rough[bi];
                    ld = sqrt(best) * M->cell;
                }
            }
        }
        if (found) {
            const double fr = isfinite(lr) ? fmax(0.0, lr) : 0.0;
            const double noise = isfinite(range) ? fmin(NOISE_MAX, NOISE_K * fmax(0.0, range)) : NOISE_MAX;
            const double extra = isfinite(ld) ? fmin(LOOKUP_TOL_MAX, LOOKUP_TOL_PER_M * fmax(0.0, ld)) : 0.0;
            double tol = BASE_TOL + ROUGH_K * fr + noise + extra;
            tol = fmin(tol, MAX_ABOVE_LOCAL);
            if (M->indoor) tol = fmin(tol, INDOOR_MAX_Z);
            const double res = p[2] - lh;
            const double nz = abs_normal_z(nrm);
            if (nrm != NULL && res > WALL_ABOVE_LOCAL && isfinite(nz) && nz < WALL_NZ_MAX) return 0;
            if (res > 0.35 && isfinite(nz) && nz < POINT_NZ_MIN) return 0;
            return res <= tol && res >= -MAX_BELOW_LOCAL;
        }
    }
    if (M->m.valid) {
        if (!isfinite(eff)) return 0;
        const double res = p[2] - eff;
        const double nz = abs_normal_z(nrm);
        if (res > 0.35 && isfinite(nz) && nz < POINT_NZ_MIN) return 0;
        const double cap = M->indoor ? INDOOR_MAX_Z : UNSUPPORTED_ABOVE;
        return res <= cap && res >= -MAX_BELOW_LOCAL;
    }
    if (!isfinite(eff)) return 0;
    return p[2] <= eff + (M->indoor ? INDOOR_MAX_Z : OUTDOOR_MAX_Z);
}

/* get_ground_mask_into (ground_seg.cpp:1137-1314) for one frame.  masks: n_returns images h x w (written whole).
 * model: the header; grids (each may be NULL; rows*cols entries, the caller learns the shape from a first call):
 * valid, obstacle, floor_z, height, roughness after pass `stop` (STAGE_FILL3 = the full model). */
void orc_ground_run(const orc_ground_frame* f, int stop, uint8_t* const* masks, orc_ground_model* model,
                    uint8_t* valid, uint8_t* obstacle, double* floor_z, double* height, double* rough) {
    const int H = f->h, W = f->w;
    for (int r = 0; r < f->n_returns; ++r)
        if (masks && masks[r]) memset(masks[r], 0, (size_t)H * W);
    Model M;
    memset(&M, 0, sizeof(M));
    M.m.fallback_z = NAN_D;
    M.cell = 0.5;
    M.inv = 2.0;
    int first = -1, last = -1;
    for (int c = 0; c < W; ++c)
        if (f->status[c] & 1u) {
            if (first < 0) first = c;
            last = c;
        }
    if (first >= 0) {
        M.m.has_columns = 1;
        build_model(f, first, last, stop, &M);
    }
    M.indoor = M.m.footprint_bound <= INDOOR_BOUND_M;
    if (model) *model = M.m;
    const size_t n = (size_t)M.m.rows * M.m.cols;
    if (M.valid) {
        if (valid) memcpy(valid, M.valid, n);
        if (obstacle) memcpy(obstacle, M.obstacle, n);
        if (floor_z) memcpy(floor_z, M.floor_z, n * sizeof(double));
        if (height) memcpy(height, M.height, n * sizeof(double));
        if (rough) memcpy(rough, M.rough, n * sizeof(double));
    }
    if (first >= 0 && masks && stop >= STAGE_FILL3) {
        const double fallback = isfinite(M.m.fallback_z) ? M.m.fallback_z : 0.0;
        double p[3];
        for (int ret = 0; ret < f->n_returns; ++ret) {
            if (!masks[ret]) continue;
            const double* nrm = ret < 2 ? f->normals[ret] : NULL;
            for (int row = 0; row < H; ++row)
                for (int col = first; col <= last; ++col) {
                    if (f->status[col] == 0u || f->range[ret][(size_t)row * W + col] == 0u) continue;
                    point_of(f, f->range[ret], row, col, p);
                    if (!finite3(p)) continue;
                    const double* nv = nrm ? nrm + ((size_t)row * W + col) * 3 : NULL;
                    if (ground_like(&M, p, norm3(p), fallback, nv)) masks[ret][(size_t)row * W + col] = 1;
                }
        }
    }
    free(M.valid), free(M.obstacle), free(M.floor_z), free(M.height), free(M.rough);
}
