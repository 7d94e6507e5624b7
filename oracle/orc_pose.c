/* orc_pose.c -- CPU oracle of pose interpolation (DESIGN f-12).  TEST INFRASTRUCTURE ONLY.
 *
 * Restates, one function per reference piece (paths relative to the reference tree):
 *   RotH::log, PoseH::log                  ouster_core/src/transform_homogeneous.cpp:31-62
 *   RotV::vee                              ouster_core/src/transform_vector.cpp:52-60
 *   PoseV::exp                             transform_vector.cpp:40-50, 96-104 -- orc_posev_exp of orc_align.c, linked
 *                                          into this library from that one source (oracle/pose.mk)
 *   Matrix3d / Matrix4d inverse            Eigen's scalar cofactor forms
 *   impl::interp_pose_range                ouster_core/include/ouster/core/pose_util.h:194-235
 *   impl::interp_pose (knot form)          pose_util.h:243-286
 *   mapping::impl::interp_pose(frame, ...) ouster_mapping/src/deskew_method.cpp:29-37
 *   impl::init_valid_column_poses          ouster_mapping/src/slam_util.cpp:129-140
 * Built with -ffp-contract=off; products sum over k in index order (DESIGN 2).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void orc_posev_exp(const double* v, double* M); /* orc_align.c */

enum { OK = 0, KNOT_ORDER = 1, ZERO_DURATION = 2, DESCENT = 3 };
enum { X_F64 = 0, X_I64 = 1 };

static double sqn3(double a, double b, double c) { return (a * a + b * b) + c * c; }

static void skew(const double* v, double a[3][3]) {
    a[0][0] = 0.0, a[0][1] = -v[2], a[0][2] = v[1];
    a[1][0] = v[2], a[1][1] = 0.0, a[1][2] = -v[0];
    a[2][0] = -v[1], a[2][1] = v[0], a[2][2] = 0.0;
}
static void mat3_mul(const double a[3][3], const double b[3][3], double c[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[i][j] = (a[i][0] * b[0][j] + a[i][1] * b[1][j]) + a[i][2] * b[2][j];
}

/* RotV::vee(angle, sin, cos) (transform_vector.cpp:52-60) */
static void rotv_vee(const double* rv, double angle, double sa, double ca, double W[3][3]) {
    if (angle < DBL_EPSILON) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) W[i][j] = i == j ? 1.0 : 0.0;
        return;
    }
    const double ax[3] = {rv[0] / angle, rv[1] / angle, rv[2] / angle};
    double a[3][3], b[3][3], bb[3][3];
    skew(ax, a);
    const double c1 = 1.0 - ca, c2 = angle - sa;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) b[i][j] = c2 * a[i][j];
    mat3_mul(b, a, bb);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) W[i][j] = ((i == j ? 1.0 : 0.0) + (c1 * a[i][j]) / angle) + bb[i][j] / angle;
}

/* Matrix3d::inverse: cofactors of column 0, det, result(i, j) = cofactor(j, i) * (1 / det) */
static double cof3(const double m[3][3], int i, int j) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1];
}
static void inverse3(const double m[3][3], double r[3][3]) {
    const double c0 = cof3(m, 0, 0), c1 = cof3(m, 1, 0), c2 = cof3(m, 2, 0);
    const double invdet = 1.0 / ((c0 * m[0][0] + c1 * m[1][0]) + c2 * m[2][0]);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[i][j] = cof3(m, j, i) * invdet;
}

/* Matrix4d::inverse (general, as PoseH::inverse): result(j, i) = (-1)^(i+j) cofactor_4x4<i, j>, / det */
static double det3_helper(const double* m, int i1, int i2, int i3, int j1, int j2, int j3) {
    return m[4 * i1 + j1] * (m[4 * i2 + j2] * m[4 * i3 + j3] - m[4 * i2 + j3] * m[4 * i3 + j2]);
}
static double cof4(const double* m, int i, int j) {
    const int i1 = (i + 1) % 4, i2 = (i + 2) % 4, i3 = (i + 3) % 4;
    const int j1 = (j + 1) % 4, j2 = (j + 2) % 4, j3 = (j + 3) % 4;
    return (det3_helper(m, i1, i2, i3, j1, j2, j3) + det3_helper(m, i2, i3, i1, j1, j2, j3)) +
           det3_helper(m, i3, i1, i2, j1, j2, j3);
}
void orc_inverse4(const double* m, double* r) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const double c = cof4(m, i, j);
            r[4 * j + i] = ((i + j) & 1) ? -c : c;
        }
    const double det = ((m[0] * r[0] + m[4] * r[1]) + m[8] * r[2]) + m[12] * r[3];
    for (int k = 0; k < 16; ++k) r[k] = r[k] / det;
}

void orc_mat4_mul(const double* a, const double* b, double* c) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            c[4 * i + j] = ((a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j]) + a[4 * i + 2] * b[8 + j]) + a[4 * i + 3] * b[12 + j];
}

/* RotH::log + PoseH::log (transform_homogeneous.cpp:31-62) */
void orc_poseh_log(const double* M, double* v) {
    double ca = 0.5 * (((M[0] + M[5]) + M[10]) - 1.0);
    ca = ca < -1.0 + DBL_EPSILON ? -1.0 + DBL_EPSILON : ca; /* std::max */
    ca = 1.0 - DBL_EPSILON < ca ? 1.0 - DBL_EPSILON : ca;   /* std::min */
    const double angle = acos(ca);
    double rv[3] = {M[9] - M[6], M[2] - M[8], M[4] - M[1]};
    const double z = sqn3(rv[0], rv[1], rv[2]);
    if (z > DBL_EPSILON) {
        const double nrm = sqrt(z);
        for (int k = 0; k < 3; ++k) rv[k] = (rv[k] / nrm) * angle;
    } else {
        for (int k = 0; k < 3; ++k) rv[k] = rv[k] / 2.0;
    }
    const double sa = sin(angle);
    double W[3][3], Wi[3][3];
    rotv_vee(rv, angle, sa, ca, W);
    inverse3(W, Wi);
    for (int i = 0; i < 3; ++i) {
        v[i] = rv[i];
        v[3 + i] = (Wi[i][0] * M[3] + Wi[i][1] * M[7]) + Wi[i][2] * M[11];
    }
}

/* x values of either dtype, read as the reference's T */
typedef union {
    double d;
    int64_t i;
} xval;
static xval xat(const void* x, int dt, size_t k) {
    xval v;
    if (dt == X_F64) v.d = ((const double*)x)[k];
    else v.i = ((const int64_t*)x)[k];
    return v;
}
static int xless(const void* x, int dt, size_t a, xval b) {
    return dt == X_F64 ? ((const double*)x)[a] < b.d : ((const int64_t*)x)[a] < b.i;
}
static int x_lt(int dt, xval a, xval b) { return dt == X_F64 ? a.d < b.d : a.i < b.i; }
static int x_ge(int dt, xval a, xval b) { return dt == X_F64 ? a.d >= b.d : a.i >= b.i; }

/* std::lower_bound as libstdc++ runs it */
static size_t lower_bound(const void* x, int dt, size_t first, size_t last, xval val) {
    size_t len = last - first;
    while (len > 0) {
        const size_t half = len >> 1, mid = first + half;
        if (xless(x, dt, mid, val)) {
            first = mid + 1;
            len = len - half - 1;
        } else {
            len = half;
        }
    }
    return first;
}

/* impl::interp_pose_range over x[b, e): err = {kind, index, -, value bits of x[index], x[index - 1]} */
static int interp_range(const void* x, int dt, size_t b, size_t e, xval t0, const double* x0, xval t1,
                        const double* x1, double* out, int64_t* err) {
    double dur_d;
    if (dt == X_F64) {
        const double duration = t1.d - t0.d;
        if (fabs(duration) < DBL_EPSILON) return ZERO_DURATION;
        dur_d = duration;
    } else {
        const int64_t duration = t1.i - t0.i; /* epsilon<int64_t> is 0: never too short */
        dur_d = (double)duration;
    }
    double ai[16], r[16], tw[6], st[6];
    orc_inverse4(x0, ai);
    orc_mat4_mul(ai, x1, r);
    orc_poseh_log(r, tw);
    const double inv = 1.0 / dur_d;
    for (int k = 0; k < 6; ++k) st[k] = inv * tw[k];
    size_t last = b;
    for (size_t j = b; j < e; ++j) {
        const xval cur = xat(x, dt, j), prev = xat(x, dt, last);
        if (x_lt(dt, cur, prev)) {
            err[1] = (int64_t)j;
            memcpy(&err[3], &cur, 8);
            memcpy(&err[4], &prev, 8);
            return DESCENT;
        }
        last = j;
        double d;
        if (dt == X_F64) d = cur.d - t0.d;
        else d = (double)(cur.i - t0.i);
        double delta[6], E[16];
        for (int k = 0; k < 6; ++k) delta[k] = d * st[k];
        orc_posev_exp(delta, E);
        orc_mat4_mul(x0, E, out + 16 * j);
    }
    return OK;
}

/* interp_pose, both forms.  poses_known: m x 16 doubles; out: n x 16, written only when the call succeeds.
 * err: 5 words (kind, index, 0, value bits of x[index], x[index - 1]).  Returns the kind. */
int orc_interp_pose(const void* x, size_t n, const void* knots, size_t m, int dt, const double* poses_known,
                    int two_pose, double* out, int64_t* err) {
    memset(err, 0, 5 * sizeof(int64_t));
    double* tmp = (double*)malloc((n ? n : 1) * 16 * sizeof(double));
    int kind = OK;
    if (two_pose) {
        kind = interp_range(x, dt, 0, n, xat(knots, dt, 0), poses_known, xat(knots, dt, 1), poses_known + 16, tmp, err);
        if (kind == ZERO_DURATION) err[1] = 0;
    } else {
        size_t curr = 0, i;
        for (i = 0; i + 1 < m && kind == OK; ++i) {
            const xval k0 = xat(knots, dt, i), k1 = xat(knots, dt, i + 1);
            if (x_ge(dt, k0, k1)) {
                kind = KNOT_ORDER;
                err[1] = (int64_t)i;
                break;
            }
            const size_t it = lower_bound(x, dt, curr, n, k1);
            if (it == curr) continue;
            kind = interp_range(x, dt, curr, it, k0, poses_known + 16 * i, k1, poses_known + 16 * (i + 1), tmp, err);
            if (kind == ZERO_DURATION) err[1] = (int64_t)i;
            curr = it;
        }
        if (kind == OK && curr < n) {
            kind = interp_range(x, dt, curr, n, xat(knots, dt, m - 2), poses_known + 16 * (m - 2),
                                xat(knots, dt, m - 1), poses_known + 16 * (m - 1), tmp, err);
            if (kind == ZERO_DURATION) err[1] = (int64_t)(m - 2);
        }
    }
    err[0] = kind;
    if (kind == OK && n) memcpy(out, tmp, n * 16 * sizeof(double));
    free(tmp);
    return kind;
}

/* ConstantVelocityDeskewMethod::update for the frames of a set (ts == NULL: empty slot), x1 == NULL:
 * init_valid_column_poses(x0).  Frames are written in slot order; the failing frame and the later ones are left
 * alone.  err: kind, column, slot, value bits. */
int orc_frames_interp_pose(const uint64_t* const* ts, const uint32_t* const* status, double* const* poses,
                           const size_t* w, size_t n_frames, double t0, const double* x0, double t1, const double* x1,
                           int64_t* err) {
    memset(err, 0, 5 * sizeof(int64_t));
    for (size_t f = 0; f < n_frames; ++f) {
        if (!ts[f]) continue;
        if (!x1) {
            for (size_t c = 0; c < w[f]; ++c)
                if (status[f][c] & 1u) memcpy(poses[f] + 16 * c, x0, 16 * sizeof(double));
            continue;
        }
        size_t nv = 0;
        size_t* cols = (size_t*)malloc((w[f] ? w[f] : 1) * sizeof(size_t));
        double* x = (double*)malloc((w[f] ? w[f] : 1) * sizeof(double));
        for (size_t c = 0; c < w[f]; ++c)
            if (status[f][c] & 1u) {
                cols[nv] = c;
                x[nv++] = (double)ts[f][c] * 1e-9;
            }
        const double knots[2] = {t0, t1};
        double pk[32];
        memcpy(pk, x0, 16 * sizeof(double));
        memcpy(pk + 16, x1, 16 * sizeof(double));
        double* out = (double*)malloc((nv ? nv : 1) * 16 * sizeof(double));
        const int kind = orc_interp_pose(x, nv, knots, 2, X_F64, pk, 1, out, err);
        if (kind == OK)
            for (size_t k = 0; k < nv; ++k) memcpy(poses[f] + 16 * cols[k], out + 16 * k, 16 * sizeof(double));
        else if (kind == DESCENT)
            err[1] = (int64_t)cols[err[1]];
        if (kind != OK) err[2] = (int64_t)f;
        free(cols);
        free(x);
        free(out);
        if (kind != OK) return kind;
    }
    return OK;
}
