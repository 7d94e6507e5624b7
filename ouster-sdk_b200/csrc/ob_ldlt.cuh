// ob_ldlt.cuh -- Eigen's 6x6 LDLT with diagonal pivoting and its solve, shared by frame-to-map ICP
// (ob_voxel_map.cu) and point-to-plane cloud alignment (ob_align.cu).
#pragma once
#include <cfloat>

#include "ob_arith.cuh"

namespace ob {
namespace {

// ---- Eigen LDLT (ldlt_inplace<Lower>::unblocked) and LDLT::_solve_impl, inner products in index order ----
// Returns info() == Success: false (NumericalIssue) when a valid pivot follows a zero one, or a zero pivot has a
// non-zero entry below it; the solution is computed either way, as Eigen's solve() does.
__device__ bool ldlt_solve6(const double* A, const double* rhs, double* x) {
    double m[6][6];
    int tr[6];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) m[i][j] = j <= i ? A[i * 6 + j] : 0.0;
    bool zero_diag = false, ok = true, found_zero = false;
    for (int k = 0; k < 6 && !zero_diag; ++k) {
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
                const double u = m[i][k];
                m[i][k] = m[big][i];
                m[big][i] = u;
            }
        }
        if (k > 0) {
            double temp[6];
            for (int j = 0; j < k; ++j) temp[j] = mul(m[j][j], m[k][j]);
            double dot = mul(m[k][0], temp[0]);
            for (int j = 1; j < k; ++j) dot = add(dot, mul(m[k][j], temp[j]));
            m[k][k] = sub(m[k][k], dot);
            for (int i = k + 1; i < 6; ++i) {
                double s = mul(m[i][0], temp[0]);
                for (int j = 1; j < k; ++j) s = add(s, mul(m[i][j], temp[j]));
                m[i][k] = sub(m[i][k], s);
            }
        }
        const double akk = m[k][k];
        const bool valid = fabs(akk) > 0.0;
        if (k == 0 && !valid) {  // the whole diagonal is zero
            for (int j = 0; j < 6; ++j) {
                tr[j] = j;
                for (int i = j + 1; i < 6; ++i) m[i][j] = 0.0;
            }
            zero_diag = true;
            break;
        }
        if (valid) {
            for (int i = k + 1; i < 6; ++i) m[i][k] = m[i][k] / akk;
        } else {
            for (int i = k + 1; i < 6; ++i) ok = ok && m[i][k] == 0.0;
        }
        if (found_zero && valid) ok = false;
        else if (!valid) found_zero = true;
    }
    for (int i = 0; i < 6; ++i) x[i] = rhs[i];
    for (int k = 0; k < 6; ++k) {
        const double s = x[k];
        x[k] = x[tr[k]];
        x[tr[k]] = s;
    }
    for (int j = 0; j < 6; ++j)
        for (int i = j + 1; i < 6; ++i) x[i] = sub(x[i], mul(x[j], m[i][j]));
    for (int i = 0; i < 6; ++i) x[i] = fabs(m[i][i]) > DBL_MIN ? x[i] / m[i][i] : 0.0;
    for (int i = 4; i >= 0; --i) {
        double s = mul(m[i + 1][i], x[i + 1]);
        for (int j = i + 2; j < 6; ++j) s = add(s, mul(m[j][i], x[j]));
        x[i] = sub(x[i], s);
    }
    for (int k = 5; k >= 0; --k) {
        const double s = x[k];
        x[k] = x[tr[k]];
        x[tr[k]] = s;
    }
    return ok;
}

}  // namespace
}  // namespace ob
