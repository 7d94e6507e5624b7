/* orc_align_clouds.c -- CPU restatement of the point-cloud align_clouds overloads (DESIGN f-14).  TEST INFRASTRUCTURE
 * ONLY: nothing under ouster-sdk_b200/ uses it.  Built by oracle/align_clouds.mk together with orc_align.c (ICP) and
 * orc_voxel.c (downsampling), with the other oracles' flags (-ffp-contract=off: no FMA).
 *
 * What it restates (reference paths relative to the reference tree, ouster-sdk 1.0.1):
 *   features of a point cloud                    ouster_algorithm/src/align_clouds.cpp:396-454, 805-882
 *   estimate_xy_footprint_bound, choose_xy_matcher_params, make_xy_grid_spec   :456-508, 892-904
 *   normalize_zero_mean_unit_norm, build_xy_bev_grid, align_xy_2d_fft          :906-1181
 *   compute_translation_histogram, best_translation_shift, align_translation_1d :1203-1298
 *   make_confidence_sample_mask, SpatialHashGridXY, xy_matching_confidence      :237-291, 1304-1477
 *   initial_pairwise_alignment                   :1496-1581
 *   align_clouds_from_features_impl and the six point-cloud overloads          :1893-1995, 2601-2651
 *
 * Order of evaluation: as orc_align.c (DESIGN 2).  Grid cells and histogram bins sum their points in row order from
 * zero; a grid's mean and squared norm sum its cells in row-major order.  The FFT is this file's own radix-2
 * decimation in time (the reference uses Eigen's kissfft, so near-tie decisions can differ from it, DESIGN 9): the
 * input in bit-reversed order, stages of length 2, 4, ..., n, butterfly u +- w v with w = twiddle(n)[j n / len],
 * twiddle(n)[k] = (cos(-2 pi k / n), sin(-2 pi k / n)), the inverse with conjugated twiddles and a final 1 / n.
 * A 2-D transform runs rows, then columns; rows known to be zero are skipped, and of the inverse only the rows the
 * shift window reads are transformed.  Neither changes a value.
 *
 * Feature order is orc_voxel.c's (voxels in order of their first row), not the reference's robin_map order. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PI_ 3.14159265358979323846
#define MIN_ICP_POINTS 20u
#define NORMAL_EPS 1e-12
#define VOXEL_SIZE_COARSE 0.4
#define TRANS_PITCH 0.2
#define NUM_TRANS 1024
#define Z_FFT_N 2048
#define MAX_Z_CORRECTION 4.0
#define XY_OVERLAP_RADIUS 0.5
#define CONF_NORMAL_DEG 5.0
#define CONF_MAX_SAMPLES 16000u
#define COARSE_STEPS 180
#define FINE_STEPS 7
#define COARSE_PIXEL 0.5
#define MIN_ENERGY 1e-10

/* orc_align.c / orc_voxel.c */
int64_t orc_cell_coord(double v, double inv);
void orc_posev_exp(const double* v, double* M);
int orc_point_to_point_align(const double* src, size_t n, const double* tgt, size_t m, const double* guess,
                             double max_corr_dist, double* out, int* iterations);
int orc_point_to_plane_align(const double* src, size_t n, const double* tgt, size_t m, const double* sn, size_t n_sn,
                             const double* tn, size_t n_tn, const double* guess, double max_corr_dist,
                             double max_normal_angle_deg, double* out, int* iterations);
size_t orc_voxel_downsample(const double* frame, size_t n, double voxel_size, double* out, uint32_t* idx_out);
int orc_voxel_downsample_xd(const double* frame, size_t n, size_t cols, double voxel_size, size_t max_pts,
                            size_t min_pts, int strategy, double* out, uint32_t* idx_out, size_t* n_out);
int orc_voxel_downsample_with_normals(const double* pts, const double* nrm, size_t n, double voxel_size,
                                      double* out_p, double* out_n, uint32_t* idx_out, size_t* n_out);

/* the layout of ob_align_clouds_trace (include/ouster_b200.h) */
typedef struct {
    size_t source_features, target_features;
    int32_t searched, coarse_index, fine_index, pad;
    double bound_m, fine_pixel_m, coarse_pixel_m, max_shift_m;
    int32_t fine_base_n, fine_fft_n, fine_max_shift, coarse_base_n, coarse_fft_n, coarse_max_shift;
    double coarse_scores[COARSE_STEPS];
    int32_t fine_z_bins[FINE_STEPS], fine_dx[FINE_STEPS], fine_dy[FINE_STEPS], pad2;
    double fine_scores[FINE_STEPS];
    double initial_pose[16];
    double icp_poses[48];
    double initial_confidence, refined_confidence;
    size_t initial_matched, initial_total, refined_matched, refined_total;
    double stage_ms[5]; /* GPU timings; 0 here */
    double* target_fine_grid;
    double* target_coarse_grid;
    double* target_z_hist;
} Trace;

int orc_align_clouds_trace_size(void) { return (int)sizeof(Trace); }

static int finite3(const double* v) { return isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]); }
static double sqn3(const double* a) { return (a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]; }
static double norm3(const double* a) { return sqrt(sqn3(a)); }
static double max_d(double a, double b) { return a < b ? b : a; }
static double min_d(double a, double b) { return b < a ? b : a; }
static void transform(const double* P, const double* p, double* x) {
    for (int d = 0; d < 3; ++d) x[d] = ((P[4 * d] * p[0] + P[4 * d + 1] * p[1]) + P[4 * d + 2] * p[2]) + P[4 * d + 3];
}
static void rotate(const double* P, const double* p, double* x) {
    for (int d = 0; d < 3; ++d) x[d] = (P[4 * d] * p[0] + P[4 * d + 1] * p[1]) + P[4 * d + 2] * p[2];
}
static void mat4_mul(const double* a, const double* b, double* c) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            c[4 * i + j] = ((a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j]) + a[4 * i + 2] * b[8 + j]) + a[4 * i + 3] * b[12 + j];
}
static int cmp_double(const void* a, const void* b) {
    const double x = *(const double*)a, y = *(const double*)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}
/* std::nth_element's value: the k-th order statistic */
static double order_stat(double* v, size_t n, size_t k) {
    qsort(v, n, sizeof(double), cmp_double);
    return v[k];
}

/* ---- features (:805-882) ---- */
typedef struct {
    double* p;   /* k x 3 */
    double* n;   /* k x 3, or NULL */
    double* dist;
    size_t k;
} Features;

static void features_free(Features* f) {
    free(f->p);
    free(f->n);
    free(f->dist);
}

static void make_features(const double* pts, const double* nrm, size_t n, Features* f) {
    memset(f, 0, sizeof(*f));
    double* vp = malloc((n + 1) * 3 * sizeof(double));
    double* vn = nrm ? malloc((n + 1) * 3 * sizeof(double)) : NULL;
    size_t k = 0;
    for (size_t i = 0; i < n; ++i) {
        const double* p = pts + 3 * i;
        if (!finite3(p)) continue;
        if (nrm) {
            const double* q = nrm + 3 * i;
            const double len = norm3(q);
            if (!finite3(q) || len <= NORMAL_EPS) continue;
            for (int d = 0; d < 3; ++d) vn[3 * k + d] = q[d] / len;
        }
        memcpy(vp + 3 * k, p, 3 * sizeof(double));
        ++k;
    }
    double* op = malloc((k + 1) * 3 * sizeof(double));
    uint32_t* idx = malloc((k + 1) * sizeof(uint32_t));
    size_t m = 0;
    if (nrm) {
        f->n = malloc((k + 1) * 3 * sizeof(double));
        orc_voxel_downsample_with_normals(vp, vn, k, VOXEL_SIZE_COARSE, op, f->n, idx, &m);
    } else if (k > 0) {
        orc_voxel_downsample_xd(vp, k, 3, VOXEL_SIZE_COARSE, 1, 1, 1 /* AVERAGE_POINT */, op, idx, &m);
        if (m == 0) { /* the reference's fallback to the valid points */
            memcpy(op, vp, k * 3 * sizeof(double));
            m = k;
        }
    }
    free(vp);
    free(vn);
    free(idx);
    f->p = op;
    f->k = m;
    f->dist = malloc((m + 1) * sizeof(double));
    for (size_t i = 0; i < m; ++i) f->dist[i] = norm3(op + 3 * i);
}

/* ---- grid parameters (:456-508, :892-904) ---- */
static double footprint(const Features* f) {
    if (f->k == 0) return 10.0;
    double* e = malloc(f->k * sizeof(double));
    for (size_t i = 0; i < f->k; ++i) e[i] = max_d(fabs(f->p[3 * i]), fabs(f->p[3 * i + 1]));
    const size_t nth = (size_t)floor(0.95 * (double)(f->k - 1));
    const double v = order_stat(e, f->k, nth);
    free(e);
    return v;
}

typedef struct {
    double pixel, bound;
    int base_n, fft_n, max_shift;
} Spec;

static Spec make_spec(double pixel, double bound, double max_shift_m) {
    Spec s;
    s.pixel = max_d(1e-6, pixel);
    s.bound = max_d(s.pixel, bound);
    const double span = 2.0 * s.bound;
    const int b = (int)ceil(span / s.pixel) + 1;
    s.base_n = b > 8 ? b : 8;
    int n = 1;
    while (n < 2 * s.base_n - 1) n <<= 1;
    s.fft_n = n > 8 ? n : 8;
    long long bins = llround(max_d(0.1, max_shift_m) / s.pixel);
    if (bins < 1) bins = 1;
    s.max_shift = (int)(bins < s.base_n / 2 ? bins : s.base_n / 2);
    return s;
}

/* ---- radix-2 FFT ---- */
static void fft(double* re, double* im, int n, int inverse, double* wr, double* wi) {
    for (int k = 0; k < n / 2; ++k) {
        const double ang = -2.0 * PI_ * (double)k / (double)n;
        wr[k] = cos(ang);
        wi[k] = inverse ? -sin(ang) : sin(ang);
    }
    for (int i = 1, j = 0; i < n; ++i) {
        int bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) {
            double t = re[i];
            re[i] = re[j];
            re[j] = t;
            t = im[i];
            im[i] = im[j];
            im[j] = t;
        }
    }
    for (int len = 2; len <= n; len <<= 1) {
        const int half = len >> 1, step = n / len;
        for (int i = 0; i < n; i += len)
            for (int j = 0; j < half; ++j) {
                const double cr = wr[j * step], ci = wi[j * step];
                const double br = re[i + j + half], bi = im[i + j + half];
                const double vr = br * cr - bi * ci, vi = br * ci + bi * cr;
                const double ur = re[i + j], ui = im[i + j];
                re[i + j] = ur + vr;
                im[i + j] = ui + vi;
                re[i + j + half] = ur - vr;
                im[i + j + half] = ui - vi;
            }
    }
    if (inverse) {
        const double s = 1.0 / (double)n;
        for (int i = 0; i < n; ++i) {
            re[i] *= s;
            im[i] *= s;
        }
    }
}

/* ---- BEV grid (:921-1019) and its normalisation (:906-919) ---- */
/* points already transformed; normals rotated (or NULL) */
static void bev_grid(const double* pts, const double* nrm, const double* dist, size_t k, const Spec* s, double* grid) {
    const int bn = s->base_n;
    memset(grid, 0, (size_t)bn * bn * sizeof(double));
    const double half = s->bound, inv = 1.0 / s->pixel;
    double min_z = DBL_MAX, max_z = -DBL_MAX;
    double* zs = malloc((k + 1) * sizeof(double));
    size_t nz = 0;
    for (size_t i = 0; i < k; ++i) {
        const double z = pts[3 * i + 2];
        if (isfinite(z)) {
            zs[nz++] = z;
            if (z < min_z) min_z = z;
            if (z > max_z) max_z = z;
        }
    }
    const double z_range = max_z - min_z;
    const int filter = isfinite(z_range) && z_range > 1.0;
    double floor_ref = min_z;
    if (filter && nz > 0) {
        size_t p = (size_t)(0.04 * (double)nz);
        if (p > nz - 1) p = nz - 1;
        floor_ref = order_stat(zs, nz, p);
    }
    free(zs);
    const double floor_cut = floor_ref + 0.2, ceil_cut = max_z - 0.1;
    for (size_t i = 0; i < k; ++i) {
        if (dist[i] <= 0.0) continue;
        const double* p = pts + 3 * i;
        if (!finite3(p)) continue;
        if (filter && (p[2] <= floor_cut || p[2] >= ceil_cut)) continue;
        if (fabs(p[0]) > half || fabs(p[1]) > half) continue;
        double w = dist[i];
        if (nrm) {
            const double* q = nrm + 3 * i;
            if (!finite3(q)) continue;
            const double strength = q[0] * q[0] + q[1] * q[1];
            if (strength < 0.5) continue;
            w *= strength;
        }
        const int ix = (int)floor((p[0] + half) * inv), iy = (int)floor((p[1] + half) * inv);
        if (ix < 0 || iy < 0 || ix >= bn || iy >= bn) continue;
        grid[(size_t)iy * bn + ix] += w;
    }
}

/* normalise in place; returns the squared sum after it (the reference's emptiness test) */
static double normalize(double* g, size_t cells) {
    double sum = 0.0;
    for (size_t i = 0; i < cells; ++i) sum += g[i];
    const double mean = sum / (double)cells;
    double nsq = 0.0;
    for (size_t i = 0; i < cells; ++i) {
        g[i] -= mean;
        nsq += g[i] * g[i];
    }
    if (!isfinite(nsq) || nsq <= 1e-30) return nsq;
    const double r = sqrt(nsq);
    double e = 0.0;
    for (size_t i = 0; i < cells; ++i) {
        g[i] /= r;
        e += g[i] * g[i];
    }
    return e;
}

/* forward 2-D spectrum of a normalised base_n^2 grid, fft_n^2 complex (re, im planes) */
static void spectrum(const double* g, const Spec* s, double* re, double* im, double* wr, double* wi) {
    const int n = s->fft_n, bn = s->base_n;
    memset(re, 0, (size_t)n * n * sizeof(double));
    memset(im, 0, (size_t)n * n * sizeof(double));
    for (int r = 0; r < bn; ++r) {
        memcpy(re + (size_t)r * n, g + (size_t)r * bn, bn * sizeof(double));
        fft(re + (size_t)r * n, im + (size_t)r * n, n, 0, wr, wi);
    }
    double* cr = malloc(2 * n * sizeof(double));
    double* ci = cr + n;
    for (int c = 0; c < n; ++c) {
        for (int r = 0; r < n; ++r) cr[r] = re[(size_t)r * n + c], ci[r] = im[(size_t)r * n + c];
        fft(cr, ci, n, 0, wr, wi);
        for (int r = 0; r < n; ++r) re[(size_t)r * n + c] = cr[r], im[(size_t)r * n + c] = ci[r];
    }
    free(cr);
}

typedef struct {
    Spec s;
    double *re, *im; /* target spectrum */
    int empty;
} TargetXY;

/* score and (dx, dy) of one moving grid against the target (:1108-1181); mg is normalised in place */
static double correlate(double* mg, const TargetXY* t, int* bdx, int* bdy, double* wr, double* wi) {
    *bdx = *bdy = 0;
    const Spec* s = &t->s;
    const int n = s->fft_n, bn = s->base_n, ms = s->max_shift;
    if (t->empty) return 0.0;
    if (normalize(mg, (size_t)bn * bn) <= MIN_ENERGY) return 0.0;
    double* re = malloc((size_t)n * n * sizeof(double));
    double* im = malloc((size_t)n * n * sizeof(double));
    spectrum(mg, s, re, im, wr, wi);
    /* columns: conj(M) T, then the inverse column transform */
    for (size_t i = 0; i < (size_t)n * n; ++i) {
        const double mr = re[i], mi = im[i], tr = t->re[i], ti = t->im[i];
        re[i] = mr * tr + mi * ti;
        im[i] = mr * ti - mi * tr;
    }
    double* cr = malloc(2 * n * sizeof(double));
    double* ci = cr + n;
    for (int c = 0; c < n; ++c) {
        for (int r = 0; r < n; ++r) cr[r] = re[(size_t)r * n + c], ci[r] = im[(size_t)r * n + c];
        fft(cr, ci, n, 1, wr, wi);
        for (int r = 0; r < n; ++r) re[(size_t)r * n + c] = cr[r], im[(size_t)r * n + c] = ci[r];
    }
    free(cr);
    double best = -DBL_MAX;
    for (int dy = -ms; dy <= ms; ++dy) {
        const int iy = dy >= 0 ? dy : n + dy;
        double* rr = re + (size_t)iy * n;
        fft(rr, im + (size_t)iy * n, n, 1, wr, wi);
        for (int dx = -ms; dx <= ms; ++dx) {
            const double v = rr[dx >= 0 ? dx : n + dx];
            if (v > best) {
                best = v;
                *bdx = dx;
                *bdy = dy;
            }
        }
    }
    free(re);
    free(im);
    return best;
}

/* ---- Z histogram (:1203-1232) and shift (:1237-1298) ---- */
static void z_hist(const double* pts, const double* nrm, const double* dist, size_t k, double* h) {
    memset(h, 0, NUM_TRANS * sizeof(double));
    for (size_t i = 0; i < k; ++i) {
        if (dist[i] <= 0.0) continue;
        const double* p = pts + 3 * i;
        double w = 1.0;
        if (nrm) {
            w = fabs(nrm[3 * i + 2]); /* |n . UnitZ| = ((n0 0 + n1 0) + n2 1) */
            if (w <= 0.5) continue;
        }
        const double z = (p[0] * 0.0 + p[1] * 0.0) + p[2] * 1.0;
        const long long pos = llround(z / TRANS_PITCH) + NUM_TRANS / 2;
        if (pos < 0 || pos >= NUM_TRANS) continue;
        h[pos] += w * dist[i];
    }
}

static int z_shift(const double* mov, const double* tgt, double* wr, double* wi) {
    double* a = calloc(4 * Z_FFT_N, sizeof(double));
    double *ar = a, *ai = a + Z_FFT_N, *br = a + 2 * Z_FFT_N, *bi = a + 3 * Z_FFT_N;
    memcpy(ar, mov, NUM_TRANS * sizeof(double));
    memcpy(br, tgt, NUM_TRANS * sizeof(double));
    fft(ar, ai, Z_FFT_N, 0, wr, wi);
    fft(br, bi, Z_FFT_N, 0, wr, wi);
    for (int i = 0; i < Z_FFT_N; ++i) {
        const double mr = ar[i], mi = ai[i], tr = br[i], ti = bi[i];
        ar[i] = mr * tr + mi * ti;
        ai[i] = mr * ti - mi * tr;
    }
    fft(ar, ai, Z_FFT_N, 1, wr, wi);
    const int ms = 20; /* min(max(1, llround(4 / 0.2)), 512) */
    int best_shift = 0;
    double best = -DBL_MAX;
    for (int s = -ms; s <= ms; ++s) {
        const double v = ar[s >= 0 ? s : Z_FFT_N + s];
        if (v > best) {
            best = v;
            best_shift = s;
        }
    }
    free(a);
    return best_shift;
}

static double z_translation(int bins) {
    return max_d(-MAX_Z_CORRECTION, min_d(TRANS_PITCH * (double)bins, MAX_Z_CORRECTION));
}

/* ---- confidence (:1304-1477) ---- */
typedef struct {
    int64_t cx, cy;
    uint32_t row;
} Cell2;
static int cmp_cell2(const void* a, const void* b) {
    const Cell2 *x = a, *y = b;
    if (x->cx != y->cx) return x->cx < y->cx ? -1 : 1;
    if (x->cy != y->cy) return x->cy < y->cy ? -1 : 1;
    return x->row < y->row ? -1 : (x->row > y->row ? 1 : 0);
}
typedef struct {
    Cell2* c;
    size_t n;
} Grid2;

static void grid2_build(Grid2* g, const double* pts, size_t k) {
    g->c = malloc((k + 1) * sizeof(Cell2));
    g->n = 0;
    for (size_t i = 0; i < k; ++i) {
        if (!finite3(pts + 3 * i)) continue;
        g->c[g->n++] = (Cell2){orc_cell_coord(pts[3 * i], 1.0 / XY_OVERLAP_RADIUS),
                               orc_cell_coord(pts[3 * i + 1], 1.0 / XY_OVERLAP_RADIUS), (uint32_t)i};
    }
    qsort(g->c, g->n, sizeof(Cell2), cmp_cell2);
}

/* first sorted position of cell (x, y) or of the next cell after it */
static size_t grid2_lower(const Grid2* g, int64_t x, int64_t y) {
    size_t lo = 0, hi = g->n;
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        const Cell2* c = g->c + mid;
        if (c->cx < x || (c->cx == x && c->cy < y)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

/* SpatialHashGridXY::nearest_xy: 9 cells in dx, dy order (int64 addition wraps), rows ascending, first strictly
 * smaller squared XY distance */
static int grid2_nearest(const Grid2* g, const double* pts, const double* q, double max_d2) {
    if (!isfinite(q[0]) || !isfinite(q[1])) return -1;
    const int64_t cx = orc_cell_coord(q[0], 1.0 / XY_OVERLAP_RADIUS), cy = orc_cell_coord(q[1], 1.0 / XY_OVERLAP_RADIUS);
    int best = -1;
    double bd = max_d2;
    for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy) {
            const int64_t x = (int64_t)((uint64_t)cx + (uint64_t)(int64_t)dx);
            const int64_t y = (int64_t)((uint64_t)cy + (uint64_t)(int64_t)dy);
            for (size_t s = grid2_lower(g, x, y); s < g->n && g->c[s].cx == x && g->c[s].cy == y; ++s) {
                const uint32_t j = g->c[s].row;
                const double ddx = pts[3 * j] - q[0], ddy = pts[3 * j + 1] - q[1];
                const double d2 = ddx * ddx + ddy * ddy;
                if (d2 < bd) {
                    bd = d2;
                    best = (int)j;
                }
            }
        }
    return best;
}

static uint8_t* sample_mask(const double* pts, size_t k) {
    if (k <= CONF_MAX_SAMPLES) return NULL;
    double* out = malloc(k * 3 * sizeof(double));
    uint32_t* idx = malloc(k * sizeof(uint32_t));
    size_t m = orc_voxel_downsample(pts, k, VOXEL_SIZE_COARSE, out, idx);
    if (m > CONF_MAX_SAMPLES) m = CONF_MAX_SAMPLES;
    uint8_t* keep = calloc(k, 1);
    for (size_t i = 0; i < m; ++i) keep[idx[i]] = 1;
    free(out);
    free(idx);
    return keep;
}

static void count_dir(const Features* q, const Features* g, const Grid2* grid, const double* R, const double* t,
                      const uint8_t* mask, int use_normals, size_t* total, size_t* matched) {
    const double cos_gate = cos(CONF_NORMAL_DEG * PI_ / 180.0);
    *total = *matched = 0;
    for (size_t i = 0; i < q->k; ++i) {
        if (mask && !mask[i]) continue;
        const double* p = q->p + 3 * i;
        if (!finite3(p)) continue;
        ++*total;
        double x[3];
        for (int d = 0; d < 3; ++d) x[d] = ((R[3 * d] * p[0] + R[3 * d + 1] * p[1]) + R[3 * d + 2] * p[2]) + t[d];
        const int nn = grid2_nearest(grid, g->p, x, XY_OVERLAP_RADIUS * XY_OVERLAP_RADIUS);
        if (nn < 0) continue;
        if (!use_normals) {
            ++*matched;
            continue;
        }
        double a[3], b[3];
        memcpy(a, q->n + 3 * i, sizeof(a));
        memcpy(b, g->n + 3 * (size_t)nn, sizeof(b));
        const double an = norm3(a), bnn = norm3(b);
        if (!(finite3(a) && finite3(b) && an > NORMAL_EPS && bnn > NORMAL_EPS)) continue;
        for (int d = 0; d < 3; ++d) {
            a[d] /= an;
            b[d] /= bnn;
        }
        double w[3];
        for (int d = 0; d < 3; ++d) w[d] = (R[3 * d] * a[0] + R[3 * d + 1] * a[1]) + R[3 * d + 2] * a[2];
        const double wsq = sqn3(w);
        if (wsq > 0.0) {
            const double wn = sqrt(wsq);
            for (int d = 0; d < 3; ++d) w[d] /= wn;
        }
        if (fabs((w[0] * b[0] + w[1] * b[1]) + w[2] * b[2]) >= cos_gate) ++*matched;
    }
}

static double confidence(const Features* s, const Features* t, const Grid2* sg, const Grid2* tg, const uint8_t* sm,
                         const uint8_t* tm, int use_normals, const double* pose, size_t* matched, size_t* total) {
    *matched = *total = 0;
    if (s->k == 0 || t->k == 0) return 0.0;
    double R[9], tr[3], Ri[9], ti[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) R[3 * i + j] = pose[4 * i + j];
        tr[i] = pose[4 * i + 3];
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Ri[3 * i + j] = R[3 * j + i];
    for (int i = 0; i < 3; ++i) ti[i] = ((-Ri[3 * i] * tr[0]) + (-Ri[3 * i + 1] * tr[1])) + (-Ri[3 * i + 2] * tr[2]);
    size_t st, sm_, tt, tm_;
    count_dir(s, t, tg, R, tr, sm, use_normals, &st, &sm_);
    count_dir(t, s, sg, Ri, ti, tm, use_normals, &tt, &tm_);
    *matched = sm_ + tm_;
    *total = st + tt;
    if (st == 0 || tt == 0) return 0.0;
    const double c = (double)(sm_ + tm_) / (double)(st + tt);
    return !isfinite(c) ? 0.0 : (c < 0.0 ? 0.0 : (c > 1.0 ? 1.0 : c));
}

/* ---- the pipeline (:1496-1581, :1893-1950) ---- */
static void candidate_pose(double yaw, const double* G, double* P) {
    const double v[6] = {0.0, 0.0, yaw, 0.0, 0.0, 0.0};
    double D[16];
    orc_posev_exp(v, D);
    D[3] = D[7] = D[11] = 0.0; /* PoseH yaw_delta; set_rot leaves the translation zero */
    mat4_mul(D, G, P);
}

/* the moving cloud at pose P: points, rotated normals */
static void apply(const Features* f, const double* P, double* x, double* n) {
    for (size_t i = 0; i < f->k; ++i) {
        transform(P, f->p + 3 * i, x + 3 * i);
        if (f->n) rotate(P, f->n + 3 * i, n + 3 * i);
    }
}

/* Returns 0, or -1 / -2 for source / target normals given without the other cloud's. */
int orc_align_clouds(const double* sp, const double* sn, size_t n, const double* tp, const double* tn, size_t m,
                     const double* guess, int compute_confidence, double* pose_out, double* conf_out, Trace* tr) {
    Trace local;
    if (!tr) tr = &local;
    double* fine_buf = tr->target_fine_grid;
    double* coarse_buf = tr->target_coarse_grid;
    double* hist_buf = tr->target_z_hist;
    memset(tr, 0, sizeof(*tr));
    tr->target_fine_grid = fine_buf;
    tr->target_coarse_grid = coarse_buf;
    tr->target_z_hist = hist_buf;
    tr->coarse_index = tr->fine_index = -1;
    if ((sn == NULL) != (tn == NULL)) return sn ? -2 : -1;
    Features S, T;
    make_features(sp, sn, n, &S);
    make_features(tp, tn, m, &T);
    tr->source_features = S.k;
    tr->target_features = T.k;
    memcpy(pose_out, guess, 16 * sizeof(double));
    *conf_out = 0.0;
    if (S.k < MIN_ICP_POINTS || T.k < MIN_ICP_POINTS) {
        features_free(&S);
        features_free(&T);
        return 0;
    }
    tr->searched = 1;
    /* project_pose_to_yaw_translation (:402-415) */
    double G[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    const double yaw0 = atan2(guess[4], guess[0]);
    const double c0 = cos(yaw0), s0 = sin(yaw0);
    G[0] = c0, G[1] = -s0, G[4] = s0, G[5] = c0;
    G[3] = guess[3], G[7] = guess[7], G[11] = guess[11];
    /* choose_xy_matcher_params(target, source, G) */
    const double fp = max_d(footprint(&T), footprint(&S));
    const double gxy = max_d(fabs(G[3]), fabs(G[7]));
    const double bound = max_d(10.0, min_d(60.0, max_d(fp, gxy) + 2.0));
    const double max_shift_m = max_d(4.0, bound);
    const double fine_pixel = bound <= 18.0 ? 0.20 : (bound <= 30.0 ? 0.15 : 0.25);
    TargetXY fine, coarse;
    fine.s = make_spec(fine_pixel, bound, max_shift_m);
    coarse.s = make_spec(COARSE_PIXEL, bound, max_shift_m);
    tr->bound_m = bound;
    tr->fine_pixel_m = fine.s.pixel;
    tr->coarse_pixel_m = coarse.s.pixel;
    tr->max_shift_m = max_shift_m;
    tr->fine_base_n = fine.s.base_n, tr->fine_fft_n = fine.s.fft_n, tr->fine_max_shift = fine.s.max_shift;
    tr->coarse_base_n = coarse.s.base_n, tr->coarse_fft_n = coarse.s.fft_n, tr->coarse_max_shift = coarse.s.max_shift;
    const int nmax = fine.s.fft_n > Z_FFT_N ? fine.s.fft_n : Z_FFT_N;
    double* wr = malloc(nmax * sizeof(double));
    double* wi = malloc(nmax * sizeof(double));
    /* target: Z histogram and both spectra, untransformed */
    double hist_t[NUM_TRANS], hist_m[NUM_TRANS];
    z_hist(T.p, T.n, T.dist, T.k, hist_t);
    if (hist_buf) memcpy(hist_buf, hist_t, sizeof(hist_t));
    TargetXY* tx[2] = {&fine, &coarse};
    double* gbuf[2] = {fine_buf, coarse_buf};
    for (int g = 0; g < 2; ++g) {
        const Spec* s = &tx[g]->s;
        const size_t cells = (size_t)s->base_n * s->base_n;
        double* grid = malloc(cells * sizeof(double));
        bev_grid(T.p, T.n, T.dist, T.k, s, grid);
        if (gbuf[g]) memcpy(gbuf[g], grid, cells * sizeof(double));
        tx[g]->re = malloc((size_t)s->fft_n * s->fft_n * sizeof(double));
        tx[g]->im = malloc((size_t)s->fft_n * s->fft_n * sizeof(double));
        tx[g]->empty = normalize(grid, cells) <= MIN_ENERGY;
        if (!tx[g]->empty) spectrum(grid, s, tx[g]->re, tx[g]->im, wr, wi);
        free(grid);
    }
    double* mx = malloc((S.k + 1) * 3 * sizeof(double));
    double* mn = S.n ? malloc((S.k + 1) * 3 * sizeof(double)) : NULL;
    double* grid = malloc((size_t)fine.s.base_n * fine.s.base_n * sizeof(double));
    /* pass 1 */
    const double coarse_step = 2.0 * PI_ / (double)COARSE_STEPS;
    double best_yaw = 0.0, best_coarse = -DBL_MAX;
    for (int yi = 0; yi < COARSE_STEPS; ++yi) {
        double P[16];
        candidate_pose((double)yi * coarse_step, G, P);
        apply(&S, P, mx, mn);
        z_hist(mx, mn, S.dist, S.k, hist_m);
        P[11] += z_translation(z_shift(hist_m, hist_t, wr, wi));
        apply(&S, P, mx, mn);
        bev_grid(mx, mn, S.dist, S.k, &coarse.s, grid);
        int dx, dy;
        tr->coarse_scores[yi] = correlate(grid, &coarse, &dx, &dy, wr, wi);
        if (tr->coarse_scores[yi] > best_coarse) {
            best_coarse = tr->coarse_scores[yi];
            best_yaw = (double)yi * coarse_step;
            tr->coarse_index = yi;
        }
    }
    /* pass 2 */
    const double half_range = 3.0 * PI_ / 180.0, step = 1.0 * PI_ / 180.0;
    double best_pose[16], best_score = -DBL_MAX;
    memcpy(best_pose, G, sizeof(G));
    for (int k = 0; k < FINE_STEPS; ++k) {
        double P[16];
        candidate_pose(best_yaw - half_range + (double)k * step, G, P);
        apply(&S, P, mx, mn);
        z_hist(mx, mn, S.dist, S.k, hist_m);
        tr->fine_z_bins[k] = z_shift(hist_m, hist_t, wr, wi);
        P[11] += z_translation(tr->fine_z_bins[k]);
        apply(&S, P, mx, mn);
        bev_grid(mx, mn, S.dist, S.k, &fine.s, grid);
        const double sc = correlate(grid, &fine, &tr->fine_dx[k], &tr->fine_dy[k], wr, wi);
        tr->fine_scores[k] = sc;
        P[3] += fine.s.pixel * (double)tr->fine_dx[k];
        P[7] += fine.s.pixel * (double)tr->fine_dy[k];
        if (sc > best_score) {
            best_score = sc;
            memcpy(best_pose, P, sizeof(P));
            tr->fine_index = k;
        }
    }
    free(mx);
    free(mn);
    free(grid);
    free(wr);
    free(wi);
    for (int g = 0; g < 2; ++g) {
        free(tx[g]->re);
        free(tx[g]->im);
    }
    memcpy(tr->initial_pose, best_pose, sizeof(best_pose));
    /* ICP (:1913-1930) */
    const int use_normals = S.n != NULL && T.n != NULL;
    const double gate = bound <= 18.0 ? 10.0 : 20.0;
    const double dists[3] = {2.0, 0.6, 0.25};
    double cur[16];
    memcpy(cur, best_pose, sizeof(cur));
    for (int p = 0; p < 3; ++p) {
        double out[16];
        int it;
        if (use_normals)
            orc_point_to_plane_align(S.p, S.k, T.p, T.k, S.n, S.k, T.n, T.k, cur, dists[p], gate, out, &it);
        else
            orc_point_to_point_align(S.p, S.k, T.p, T.k, cur, dists[p], out, &it);
        memcpy(cur, out, sizeof(cur));
        memcpy(tr->icp_poses + 16 * p, cur, sizeof(cur));
    }
    /* confidence and the guard (:1932-1949) */
    Grid2 sg, tg;
    grid2_build(&sg, S.p, S.k);
    grid2_build(&tg, T.p, T.k);
    uint8_t* smask = sample_mask(S.p, S.k);
    uint8_t* tmask = sample_mask(T.p, T.k);
    const double ci = confidence(&S, &T, &sg, &tg, smask, tmask, use_normals, best_pose, &tr->initial_matched,
                                 &tr->initial_total);
    double cr = confidence(&S, &T, &sg, &tg, smask, tmask, use_normals, cur, &tr->refined_matched, &tr->refined_total);
    tr->initial_confidence = ci;
    tr->refined_confidence = cr;
    if (cr + 1e-6 < ci) {
        memcpy(cur, best_pose, sizeof(cur));
        cr = ci;
    }
    memcpy(pose_out, cur, sizeof(cur));
    *conf_out = compute_confidence ? cr : 0.0;
    free(smask);
    free(tmask);
    free(sg.c);
    free(tg.c);
    features_free(&S);
    features_free(&T);
    return 0;
}

/* xy_matching_confidence alone, for given features (rows as the features) and pose: to check the GPU's counts at
 * the GPU's poses.  Returns the confidence; matched / total are the two directions' sums. */
double orc_align_clouds_confidence(const double* sp, const double* sn, size_t n, const double* tp, const double* tn,
                                   size_t m, const double* pose, size_t* matched, size_t* total) {
    Features S = {(double*)sp, (double*)sn, NULL, n}, T = {(double*)tp, (double*)tn, NULL, m};
    Grid2 sg, tg;
    grid2_build(&sg, sp, n);
    grid2_build(&tg, tp, m);
    uint8_t* smask = sample_mask(sp, n);
    uint8_t* tmask = sample_mask(tp, m);
    const double c = confidence(&S, &T, &sg, &tg, smask, tmask, sn && tn, pose, matched, total);
    free(smask);
    free(tmask);
    free(sg.c);
    free(tg.c);
    return c;
}

/* the features of one cloud (for tests): returns the count; out_p / out_n hold n rows */
size_t orc_align_clouds_features(const double* pts, const double* nrm, size_t n, double* out_p, double* out_n) {
    Features f;
    make_features(pts, nrm, n, &f);
    memcpy(out_p, f.p, f.k * 3 * sizeof(double));
    if (nrm) memcpy(out_n, f.n, f.k * 3 * sizeof(double));
    const size_t k = f.k;
    features_free(&f);
    return k;
}
