// ob_se3.cuh -- SE(3) pieces in pinned double arithmetic, shared by cloud-to-cloud ICP (ob_align.cu), global cloud
// alignment (ob_align_clouds.cu) and pose interpolation (ob_pose_interp.cu): PoseV::exp, PoseH::log, the 3 x 3 and
// 4 x 4 inverses, the 4 x 4 product and a 4 x 4 pose applied to a point or a direction.
//
// What it restates (reference paths relative to the reference tree):
//   PoseV::exp, RotV::exp, RotV::vee          ouster_core/src/transform_vector.cpp:40-60, 96-104
//   RotH::log, PoseH::log                     ouster_core/src/transform_homogeneous.cpp:31-62
//   Eigen Matrix3d::inverse, Matrix4d::inverse  the scalar cofactor forms (InverseImpl.h)
//
// Every product and sum goes through __d*_rn, so nvcc cannot contract it into an FMA, and products sum over k in
// index order (DESIGN 2).  The CPU oracle (oracle/orc_align.c, oracle/orc_pose.c) states the same operations.
#pragma once
#include <cfloat>

#include "ob_arith.cuh"

namespace ob {
namespace {

__device__ void mat3_mul(const double a[3][3], const double b[3][3], double c[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[i][j] = add(add(mul(a[i][0], b[0][j]), mul(a[i][1], b[1][j])), mul(a[i][2], b[2][j]));
}
__device__ void skew(const double* v, double a[3][3]) {
    a[0][0] = 0.0, a[0][1] = -v[2], a[0][2] = v[1];
    a[1][0] = v[2], a[1][1] = 0.0, a[1][2] = -v[0];
    a[2][0] = -v[1], a[2][1] = v[0], a[2][2] = 0.0;
}

// ---- PoseV::exp (transform_vector.cpp:40-60, 96-104): v = (rotation vector, translation) -> row-major 4 x 4 ----
__device__ void posev_exp(const double* v, double* M) {
    const double numeric_eps = 1.4901161193847656e-08;  // sqrt(DBL_EPSILON)
    const double angle = norm3(v);
    const double sa = sin(angle), ca = cos(angle);
    double R[3][3], V[3][3];
    const double ax[3] = {v[0] / angle, v[1] / angle, v[2] / angle};
    double a[3][3], b[3][3], bb[3][3];
    if (angle < numeric_eps) {  // I + skew(v)
        skew(v, a);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i][j] = add(i == j ? 1.0 : 0.0, a[i][j]);
    } else {  // I + sin A + ((1 - cos) A) A, A = skew(v / angle)
        skew(ax, a);
        const double c1 = sub(1.0, ca);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) b[i][j] = mul(c1, a[i][j]);
        mat3_mul(b, a, bb);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i][j] = add(add(i == j ? 1.0 : 0.0, mul(sa, a[i][j])), bb[i][j]);
    }
    if (angle < DBL_EPSILON) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) V[i][j] = i == j ? 1.0 : 0.0;
    } else {  // I + ((1 - cos) A) / angle + (((angle - sin) A) A) / angle
        skew(ax, a);
        const double c1 = sub(1.0, ca), c2 = sub(angle, sa);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) b[i][j] = mul(c2, a[i][j]);
        mat3_mul(b, a, bb);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                V[i][j] = add(add(i == j ? 1.0 : 0.0, mul(c1, a[i][j]) / angle), bb[i][j] / angle);
    }
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) M[4 * i + j] = R[i][j];
        M[4 * i + 3] = add(add(mul(V[i][0], v[3]), mul(V[i][1], v[4])), mul(V[i][2], v[5]));
    }
    M[12] = M[13] = M[14] = 0.0;
    M[15] = 1.0;
}

// ---- Eigen's Matrix3d::inverse: cofactors of column 0, det = their dot with column 0, result(i, j) =
// cofactor(j, i) * (1 / det) ----
__device__ __forceinline__ double cof3(const double m[3][3], int i, int j) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return sub(mul(m[i1][j1], m[i2][j2]), mul(m[i1][j2], m[i2][j1]));
}
__device__ void inverse3(const double m[3][3], double r[3][3]) {
    const double c0 = cof3(m, 0, 0), c1 = cof3(m, 1, 0), c2 = cof3(m, 2, 0);
    const double invdet = 1.0 / add(add(mul(c0, m[0][0]), mul(c1, m[1][0])), mul(c2, m[2][0]));
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[i][j] = mul(cof3(m, j, i), invdet);
}

// ---- Eigen's general Matrix4d::inverse (PoseH::inverse is not a rigid inverse), scalar cofactor form:
// result(j, i) = (-1)^(i+j) cofactor_4x4<i, j>, then every entry / (column 0 . row 0 of the result) ----
__device__ __forceinline__ double det3_helper(const double* m, int i1, int i2, int i3, int j1, int j2, int j3) {
    return mul(m[4 * i1 + j1], sub(mul(m[4 * i2 + j2], m[4 * i3 + j3]), mul(m[4 * i2 + j3], m[4 * i3 + j2])));
}
__device__ __forceinline__ double cof4(const double* m, int i, int j) {
    const int i1 = (i + 1) % 4, i2 = (i + 2) % 4, i3 = (i + 3) % 4;
    const int j1 = (j + 1) % 4, j2 = (j + 2) % 4, j3 = (j + 3) % 4;
    return add(add(det3_helper(m, i1, i2, i3, j1, j2, j3), det3_helper(m, i2, i3, i1, j1, j2, j3)),
               det3_helper(m, i3, i1, i2, j1, j2, j3));
}
__device__ void inverse4(const double* m, double* r) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const double c = cof4(m, i, j);
            r[4 * j + i] = ((i + j) & 1) ? -c : c;
        }
    const double det = add(add(add(mul(m[0], r[0]), mul(m[4], r[1])), mul(m[8], r[2])), mul(m[12], r[3]));
    for (int k = 0; k < 16; ++k) r[k] = r[k] / det;
}

// c = a * b, row-major 4 x 4
__device__ __forceinline__ void mat4_mul(const double* a, const double* b, double* c) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            c[4 * i + j] = add(add(add(mul(a[4 * i], b[j]), mul(a[4 * i + 1], b[4 + j])), mul(a[4 * i + 2], b[8 + j])),
                               mul(a[4 * i + 3], b[12 + j]));
}

// x = R p + t and x = R p for the top 3 x 4 of a row-major pose, summed left to right: ((r0 p0 + r1 p1) + r2 p2) + t.
// ob_project.cuh's pose_row sums the dewarp's order, r0 p0 + (r1 p1 + r2 p2), instead.
__device__ __forceinline__ void mat4_transform(const double* P, const double* p, double* x) {
    for (int d = 0; d < 3; ++d)
        x[d] = add(add(add(mul(P[4 * d], p[0]), mul(P[4 * d + 1], p[1])), mul(P[4 * d + 2], p[2])), P[4 * d + 3]);
}
__device__ __forceinline__ void mat4_rotate(const double* P, const double* p, double* x) {
    for (int d = 0; d < 3; ++d) x[d] = add(add(mul(P[4 * d], p[0]), mul(P[4 * d + 1], p[1])), mul(P[4 * d + 2], p[2]));
}

// ---- PoseH::log (transform_homogeneous.cpp:31-62): row-major 4 x 4 -> v = (rotation vector, translation) ----
__device__ void poseh_log(const double* M, double* v) {
    double ca = mul(0.5, sub(add(add(M[0], M[5]), M[10]), 1.0));
    const double lo = -1.0 + DBL_EPSILON, hi = 1.0 - DBL_EPSILON;
    ca = ca < lo ? lo : ca;  // std::max(ca, -1 + EPS)
    ca = hi < ca ? hi : ca;  // std::min(ca, 1 - EPS)
    const double angle = acos(ca);
    double rv[3] = {sub(M[9], M[6]), sub(M[2], M[8]), sub(M[4], M[1])};
    const double z = sqn3(rv[0], rv[1], rv[2]);
    if (z > DBL_EPSILON) {
        const double nrm = sqrt(z);  // normalize(): /= sqrt(squaredNorm)
        for (int k = 0; k < 3; ++k) rv[k] = mul(rv[k] / nrm, angle);
    } else {
        for (int k = 0; k < 3; ++k) rv[k] = rv[k] / 2.0;
    }
    const double sa = sin(angle);
    double W[3][3];  // RotV::vee(angle, sin, cos) of the rotation vector
    if (angle < DBL_EPSILON) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) W[i][j] = i == j ? 1.0 : 0.0;
    } else {
        const double ax[3] = {rv[0] / angle, rv[1] / angle, rv[2] / angle};
        double a[3][3], b[3][3], bb[3][3];
        skew(ax, a);
        const double c1 = sub(1.0, ca), c2 = sub(angle, sa);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) b[i][j] = mul(c2, a[i][j]);
        mat3_mul(b, a, bb);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                W[i][j] = add(add(i == j ? 1.0 : 0.0, mul(c1, a[i][j]) / angle), bb[i][j] / angle);
    }
    double Wi[3][3];
    inverse3(W, Wi);
    for (int i = 0; i < 3; ++i) {
        v[i] = rv[i];
        v[3 + i] = add(add(mul(Wi[i][0], M[3]), mul(Wi[i][1], M[7])), mul(Wi[i][2], M[11]));
    }
}

}  // namespace
}  // namespace ob
