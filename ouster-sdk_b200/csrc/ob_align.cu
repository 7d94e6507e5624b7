// ob_align.cu -- cloud-to-cloud ICP (DESIGN f-7): algorithm::point_to_point_align / point_to_plane_align and the
// SpatialHashGrid3D nearest-neighbour search they run on.
//
// What it replaces (reference paths relative to the reference tree, ouster-sdk 1.0.1):
//   median_abs, SpatialHashGrid3D                ouster_algorithm/src/align_clouds.cpp:146-235
//   cell of a point, 27-cell order               ouster_algorithm/include/ouster/algorithm/impl/spatial_hash.h:73-101
//   point_to_point_align                         align_clouds.cpp:1590-1722
//   point_to_plane_align                         align_clouds.cpp:1724-1874
//   PoseV::exp (RotV::exp, RotV::vee)            ouster_core/src/transform_vector.cpp:40-60, 96-104
//   Eigen JacobiSVD<Matrix3d>, LDLT<Matrix<double, 6, 6>>
//
// Grid, once per call: int64 cell keys (x86 cvttsd2si: NaN / out of range -> INT64_MIN), a stable radix sort of
// (pad, x, y, z; row) so a cell's rows stay in ascending order, and an open-addressing table from cell to its
// [begin, end) of sorted positions.  Rows the reference leaves out of the grid get the pad bit and sort last.
//
// Per iteration, all on the stream, every kernel returning at once once the device-side `done` flag is set:
//   association   one thread per source row: transform, 27-cell search, gates, residual; a valid flag, the row's
//                 pair and the key |r| (or a pad key) for the median;
//   compaction    order-preserving, so the pairs are in source-row order as the reference's vector; the count
//                 stays on the device;
//   median        a CUB radix sort of the |r| keys (non-negative doubles order as their bits), over the capacity;
//   sums          fixed-shape trees: leaves of kLeaf consecutive pairs summed in order, then pairwise up to the
//                 root; the shape depends on the pair count only, so replays give identical bits;
//   solve         one block: the root, then thread 0 runs the SVD (point-to-point) or the LDLT and PoseV::exp
//                 (point-to-plane), composes the pose and sets the stop flag.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cuda/std/tuple>

#include <algorithm>
#include <cfloat>
#include <cmath>

#include "ob_api_common.h"
#include "ob_cub.cuh"
#include "ob_ldlt.cuh"
#include "ob_rows.cuh"
#include "ob_se3.cuh"
#include "ob_voxel_common.cuh"

namespace ob {
namespace {

constexpr unsigned long long kMinIcpPoints = 20;  // MIN_ICP_POINTS, align_clouds.cpp:308
constexpr int kMaxIterations = 10;                // icp_max_iterations
constexpr double kNormalEps = 1e-12;              // NORMAL_EPS
constexpr int kJacobiMaxSweeps = 64;              // a guard only: a 3x3 converges in a handful of sweeps
constexpr unsigned kThreads = 256;
constexpr unsigned kLeaf = 32;                    // pairs per leaf of the summation tree
constexpr unsigned kTreeThreads = 256;
constexpr unsigned long long kPadKey = ~0ull;     // sorts after every |r|
constexpr int kPair = 7;                          // x (3), q or n_tgt (3), r

// ---- SpatialHashGrid3D ----
struct GKey {
    uint32_t pad;  // 1: not in the grid (row >= n, non-finite, or a bad normal); sorts after every cell
    int64_t x, y, z;
};
struct GKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, int64_t&, int64_t&, int64_t&> operator()(GKey& k) const {
        return {k.pad, k.x, k.y, k.z};
    }
};
constexpr int kGKeyBits = 193;  // x, y, z and the low bit of pad

__device__ __forceinline__ bool same_cell(const GKey& a, const GKey& b) {
    return a.pad == b.pad && a.x == b.x && a.y == b.y && a.z == b.z;
}
__device__ __forceinline__ unsigned cell_slot(int64_t x, int64_t y, int64_t z, unsigned mask) {
    unsigned long long h = static_cast<unsigned long long>(x) * 0x9E3779B97F4A7C15ull;
    h ^= static_cast<unsigned long long>(y) * 0xC2B2AE3D27D4EB4Full;
    h ^= static_cast<unsigned long long>(z) * 0x165667B19E3779F9ull;
    h ^= h >> 32;
    h *= 0xD6E8FEB86659FD93ull;
    h ^= h >> 32;
    return static_cast<unsigned>(h) & mask;
}

struct Grid {
    const int64_t* ckey;   // cell x 3
    const uint32_t* cbeg;  // cell -> first sorted position
    const uint32_t* cend;  // cell -> one past its last
    const int32_t* table;  // slot -> cell, or -1
    unsigned mask;
    const double* pts;     // sorted position x 3
    const uint32_t* row;   // sorted position -> target row
    double inv;            // 1 / cell_size
};

template <typename T>
__global__ void gr_key_kernel(Rows t, const void* normals, double inv, GKey* keys, uint32_t* seq) {
    const unsigned i = tid_global();
    if (i >= t.cap) return;
    GKey k{1u, 0, 0, 0};
    if (i < rows_n(t)) {
        double p[3];
        load3<T>(t.p, i, p);
        bool ok = finite3(p);
        if (ok && normals) {  // the point-to-plane constructor, align_clouds.cpp:195
            double nn[3];
            load3<T>(normals, i, nn);
            ok = finite3(nn) && norm3(nn) > kNormalEps;
        }
        if (ok)
            k = GKey{0u, floor_cast<int64_t>(mul(p[0], inv)), floor_cast<int64_t>(mul(p[1], inv)),
                     floor_cast<int64_t>(mul(p[2], inv))};
    }
    keys[i] = k;
    seq[i] = i;
}

__global__ void gr_head_kernel(unsigned cap, const GKey* sk, uint32_t* head) {
    const unsigned q = tid_global();
    if (q >= cap) return;
    head[q] = (sk[q].pad == 0u && (q == 0 || !same_cell(sk[q], sk[q - 1]))) ? 1u : 0u;
}

// cells (numbered by the inclusive scan of the heads), their ranges and table slots; the points in sorted order
template <typename T>
__global__ void gr_fill_kernel(unsigned cap, const void* tgt, const GKey* sk, const uint32_t* sseq, const uint32_t* cid,
                               int64_t* ckey, uint32_t* cbeg, uint32_t* cend, int32_t* table, unsigned mask,
                               double* pts, uint32_t* row) {
    const unsigned q = tid_global();
    if (q >= cap) return;
    const GKey k = sk[q];
    if (k.pad) return;
    const unsigned c = cid[q] - 1;
    load3<T>(tgt, sseq[q], pts + 3 * static_cast<size_t>(q));
    row[q] = sseq[q];
    if (q == 0 || !same_cell(k, sk[q - 1])) {
        ckey[3 * c] = k.x;
        ckey[3 * c + 1] = k.y;
        ckey[3 * c + 2] = k.z;
        cbeg[c] = q;
        unsigned s = cell_slot(k.x, k.y, k.z, mask);
        while (atomicCAS(table + s, -1, static_cast<int>(c)) != -1) s = (s + 1) & mask;
    }
    if (q + 1 == cap || !same_cell(k, sk[q + 1])) cend[c] = q + 1;
}

__device__ __forceinline__ int grid_find(const Grid& g, int64_t x, int64_t y, int64_t z) {
    for (unsigned s = cell_slot(x, y, z, g.mask);; s = (s + 1) & g.mask) {  // the table is at most half full
        const int c = g.table[s];
        if (c < 0) return -1;
        if (g.ckey[3 * c] == x && g.ckey[3 * c + 1] == y && g.ckey[3 * c + 2] == z) return c;
    }
}

// SpatialHashGrid3D::nearest (align_clouds.cpp:203-226): the 27 cells in dx, dy, dz order (int64 addition wraps),
// a cell's rows in ascending index, the first strictly smaller squared distance kept
__device__ int grid_nearest(const Grid& g, const double* q, double max_dist_sq) {
    if (!finite3(q) || !isfinite(max_dist_sq) || max_dist_sq <= 0.0) return -1;
    const int64_t c[3] = {floor_cast<int64_t>(mul(q[0], g.inv)), floor_cast<int64_t>(mul(q[1], g.inv)),
                          floor_cast<int64_t>(mul(q[2], g.inv))};
    int best = -1;
    double best_d2 = max_dist_sq;
    for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy)
            for (int dz = -1; dz <= 1; ++dz) {
                const int cell = grid_find(g, static_cast<int64_t>(static_cast<unsigned long long>(c[0]) + dx),
                                           static_cast<int64_t>(static_cast<unsigned long long>(c[1]) + dy),
                                           static_cast<int64_t>(static_cast<unsigned long long>(c[2]) + dz));
                if (cell < 0) continue;
                const unsigned e = g.cend[cell];
                for (unsigned s = g.cbeg[cell]; s < e; ++s) {
                    const double* p = g.pts + 3 * static_cast<size_t>(s);
                    const double d2 = sqn3(sub(p[0], q[0]), sub(p[1], q[1]), sub(p[2], q[2]));
                    if (d2 < best_d2) {
                        best_d2 = d2;
                        best = static_cast<int>(g.row[s]);
                    }
                }
            }
    return best;
}

template <typename T>
__global__ void al_nearest_kernel(Rows q, Grid g, double max_dist_sq, int32_t* out) {
    const unsigned i = tid_global();
    if (i >= q.cap || i >= rows_n(q)) return;
    double p[3];
    load3<T>(q.p, i, p);
    out[i] = grid_nearest(g, p, max_dist_sq);
}

// ---- small dense pieces (DESIGN 2: products sum over k in index order, norms are sqrt of sqn3) ----
// a = b * a, row-major 4 x 4 (PoseH(delta) * current_pose)
__device__ void pose_premul(const double* b, double* a) {
    double r[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            r[4 * i + j] = add(add(add(mul(b[4 * i], a[j]), mul(b[4 * i + 1], a[4 + j])), mul(b[4 * i + 2], a[8 + j])),
                               mul(b[4 * i + 3], a[12 + j]));
    for (int j = 0; j < 16; ++j) a[j] = r[j];
}
// ---- Eigen 3.4 JacobiSVD<Matrix3d>(A, ComputeFullU | ComputeFullV) ----
// two-sided Jacobi sweeps with real_2x2_jacobi_svd and JacobiRotation::makeJacobi, then |diagonal| (U's column
// negated for a negative entry), rescaled and sorted decreasing; false for a non-finite input (InvalidInput)
__device__ void make_jacobi(double x, double y, double z, double* c, double* s) {
    const double deno = mul(2.0, fabs(y));
    if (deno < DBL_MIN) {
        *c = 1.0;
        *s = 0.0;
        return;
    }
    const double tau = sub(x, z) / deno;
    const double w = sqrt(add(mul(tau, tau), 1.0));
    const double t = tau > 0.0 ? 1.0 / add(tau, w) : 1.0 / sub(tau, w);
    const double sign_t = t > 0.0 ? 1.0 : -1.0;
    const double n = 1.0 / sqrt(add(mul(t, t), 1.0));
    *s = mul(mul(mul(-sign_t, y / fabs(y)), fabs(t)), n);
    *c = n;
}
// apply_rotation_in_the_plane: x' = c x + s y, y' = -s x + c y
__device__ void rot_rows(double m[3][3], int p, int q, double c, double s) {
    for (int j = 0; j < 3; ++j) {
        const double xi = m[p][j], yi = m[q][j];
        m[p][j] = add(mul(c, xi), mul(s, yi));
        m[q][j] = add(mul(-s, xi), mul(c, yi));
    }
}
__device__ void rot_cols(double m[3][3], int p, int q, double c, double s) {
    for (int i = 0; i < 3; ++i) {
        const double xi = m[i][p], yi = m[i][q];
        m[i][p] = add(mul(c, xi), mul(s, yi));
        m[i][q] = add(mul(-s, xi), mul(c, yi));
    }
}
__device__ bool svd3(const double* A, double u[3][3], double v[3][3]) {
    double scale = 0.0;
    for (int i = 0; i < 9; ++i) {
        const double a = fabs(A[i]);
        if (isnan(a)) return false;
        if (a > scale) scale = a;
    }
    if (!isfinite(scale)) return false;
    if (scale == 0.0) scale = 1.0;
    double w[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            w[i][j] = A[3 * i + j] / scale;
            u[i][j] = v[i][j] = i == j ? 1.0 : 0.0;
        }
    const double precision = mul(2.0, DBL_EPSILON);
    double max_diag = smax(smax(fabs(w[0][0]), fabs(w[1][1])), fabs(w[2][2]));
    bool finished = false;
    for (int sweep = 0; !finished && sweep < kJacobiMaxSweeps; ++sweep) {
        finished = true;
        for (int p = 1; p < 3; ++p)
            for (int q = 0; q < p; ++q) {
                const double threshold = smax(DBL_MIN, mul(precision, max_diag));
                if (!(fabs(w[p][q]) > threshold || fabs(w[q][p]) > threshold)) continue;
                finished = false;
                const double m00 = w[p][p], m01 = w[p][q], m10 = w[q][p], m11 = w[q][q];
                const double t = add(m00, m11), d = sub(m10, m01);
                double c1, s1;
                if (fabs(d) < DBL_MIN) {
                    s1 = 0.0;
                    c1 = 1.0;
                } else {
                    const double uu = t / d;
                    const double tmp = sqrt(add(1.0, mul(uu, uu)));
                    s1 = 1.0 / tmp;
                    c1 = uu / tmp;
                }
                const double n00 = add(mul(c1, m00), mul(s1, m10)), n01 = add(mul(c1, m01), mul(s1, m11));
                const double n11 = add(mul(-s1, m01), mul(c1, m11));
                double cr, sr;
                make_jacobi(n00, n01, n11, &cr, &sr);
                const double cl = sub(mul(c1, cr), mul(s1, -sr)), sl = add(mul(c1, -sr), mul(s1, cr));
                rot_rows(w, p, q, cl, sl);
                rot_cols(u, p, q, cl, sl);
                rot_cols(w, p, q, cr, -sr);
                rot_cols(v, p, q, cr, -sr);
                max_diag = smax(max_diag, smax(fabs(w[p][p]), fabs(w[q][q])));
            }
    }
    double s[3];
    for (int i = 0; i < 3; ++i) {
        const double a = w[i][i];
        s[i] = fabs(a);
        if (a < 0.0)
            for (int r = 0; r < 3; ++r) u[r][i] = -u[r][i];
    }
    for (int i = 0; i < 3; ++i) s[i] = mul(s[i], scale);
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
    return true;
}

// ---- the iteration ----
struct AlignState {
    double pose[16];   // current_pose
    double guess[16];  // initial_guess
    double cx[3], cq[3];
    unsigned long long n_pairs;
    int done;        // a break was taken (or the clouds are too small)
    int solved_any;  // solved_any_level
    int iterations;  // iterations that reached the solve
    int pad;
};

__global__ void al_init_kernel(Rows s, Rows t, const double* guess, AlignState* st) {
    AlignState z{};
    for (int j = 0; j < 16; ++j) z.guess[j] = z.pose[j] = guess ? guess[j] : (j % 5 == 0 ? 1.0 : 0.0);
    z.done = (rows_n(s) < kMinIcpPoints || rows_n(t) < kMinIcpPoints) ? 1 : 0;
    *st = z;
}

// one thread per source row (align_clouds.cpp:1626-1642, 1781-1814): the pair, its valid flag and its |r| key
template <typename T, bool kPlane>
__global__ void al_assoc_kernel(Rows src, const void* snrm, const void* tgt, const void* tnrm, Grid g, double max_d2,
                                double cos_gate, unsigned kcap, const AlignState* st, double* rows,
                                uint32_t* valid, uint32_t* block_count, unsigned long long* keys) {
    if (st->done) return;
    const unsigned i = tid_global();
    bool ok = false;
    double r = 0.0;
    if (i < rows_n(src)) {
        const double* P = st->pose;
        double p[3], ns[3];
        load3<T>(src.p, i, p);
        bool use = true;
        if (kPlane) {
            load3<T>(snrm, i, ns);
            const double nn = norm3(ns);
            use = finite3(ns) && nn > kNormalEps;
            for (int d = 0; d < 3; ++d) ns[d] = ns[d] / nn;
        }
        if (use) {
            double x[3];
            mat4_transform(P, p, x);
            const int j = grid_nearest(g, x, max_d2);
            if (j >= 0) {
                double q[3], v[3];
                load3<T>(tgt, j, q);
                const double dv[3] = {sub(x[0], q[0]), sub(x[1], q[1]), sub(x[2], q[2])};
                if (!kPlane) {
                    r = norm3(dv);
                    ok = finite3(x) && finite3(q) && isfinite(r);
                    for (int d = 0; d < 3; ++d) v[d] = q[d];
                } else {
                    double nw[3];
                    mat4_rotate(P, ns, nw);
                    load3<T>(tnrm, j, v);
                    const double tn = norm3(v);
                    if (finite3(v) && tn > kNormalEps) {
                        for (int d = 0; d < 3; ++d) v[d] = v[d] / tn;
                        const double n_align = fabs(dot3(v, nw));
                        if (isfinite(n_align) && !(n_align < cos_gate)) {
                            r = dot3(v, dv);
                            ok = isfinite(r);
                        }
                    }
                }
                if (ok) {
                    double* o = rows + static_cast<size_t>(kPair) * i;
                    for (int d = 0; d < 3; ++d) {
                        o[d] = x[d];
                        o[3 + d] = v[d];
                    }
                    o[6] = r;
                }
            }
        }
    }
    if (i < kcap) {
        valid[i] = ok ? 1u : 0u;
        keys[i] = ok ? static_cast<unsigned long long>(__double_as_longlong(fabs(r))) : kPadKey;
    }
    const int c = __syncthreads_count(ok);
    if (threadIdx.x == 0) block_count[blockIdx.x] = static_cast<uint32_t>(c);
}

// order-preserving compaction of the valid pairs; the last block writes the pair count
__global__ void al_compact_kernel(unsigned kcap, const double* rows, const uint32_t* valid, const uint32_t* block_count,
                                  double* pairs, AlignState* st) {
    if (st->done) return;
    compact_rows<kThreads>(kcap, valid, block_count, &st->n_pairs, [&](unsigned i, size_t o) {
        for (int d = 0; d < kPair; ++d) pairs[kPair * o + d] = rows[kPair * static_cast<size_t>(i) + d];
    });
}

// median_abs over the sorted keys, then the MAD-scaled Huber threshold (align_clouds.cpp:1650-1655)
__device__ double huber_delta(unsigned long long n, const unsigned long long* skeys, double max_corr_dist) {
    const unsigned long long mid = n / 2;
    const double hi = __longlong_as_double(static_cast<long long>(skeys[mid]));
    const double mad = (n & 1ull) ? hi : mul(0.5, add(__longlong_as_double(static_cast<long long>(skeys[mid - 1])), hi));
    double sigma = mul(1.4826, mad);
    if (!isfinite(sigma) || sigma < 1e-4) sigma = smax(1e-3, mul(0.25, max_corr_dist));
    return mul(1.5, sigma);
}
__device__ __forceinline__ double huber_w(double r, double delta) {
    const double abs_r = fabs(r);
    return (abs_r <= delta || delta <= 0.0) ? 1.0 : delta / abs_r;
}

enum : int { kCentroid = 0, kCovariance = 1, kPlaneSystem = 2 };
template <int kKind>
struct Width;
template <>
struct Width<kCentroid> {
    static constexpr int value = 7;  // w, w x, w q
};
template <>
struct Width<kCovariance> {
    static constexpr int value = 9;  // (w (x - c_x)) (q - c_q)^T, row-major
};
template <>
struct Width<kPlaneSystem> {
    static constexpr int value = 27;  // H lower triangle row by row (21), b (6)
};

// one thread per leaf: pairs [kLeaf j, kLeaf (j + 1)) summed from zero in order
template <int kKind>
__global__ void al_leaf_kernel(const double* pairs, const unsigned long long* skeys, double max_corr_dist,
                               const AlignState* st, unsigned slots, double* val) {
    constexpr int K = Width<kKind>::value;
    if (st->done) return;
    const unsigned long long n = st->n_pairs;
    const unsigned j = tid_global();
    const unsigned long long b = static_cast<unsigned long long>(j) * kLeaf;
    if (n < kMinIcpPoints || j >= slots || b >= n) return;
    const unsigned long long e = min(b + kLeaf, n);
    const double delta = huber_delta(n, skeys, max_corr_dist);
    double acc[K];
    for (int k = 0; k < K; ++k) acc[k] = 0.0;
    for (unsigned long long i = b; i < e; ++i) {
        const double* c = pairs + kPair * i;
        const double w = huber_w(c[6], delta);
        if (kKind == kCentroid) {
            acc[0] = add(acc[0], w);
            for (int d = 0; d < 3; ++d) {
                acc[1 + d] = add(acc[1 + d], mul(w, c[d]));
                acc[4 + d] = add(acc[4 + d], mul(w, c[3 + d]));
            }
        } else if (kKind == kCovariance) {
            double a[3], q[3];
            for (int d = 0; d < 3; ++d) {
                a[d] = mul(w, sub(c[d], st->cx[d]));
                q[d] = sub(c[3 + d], st->cq[d]);
            }
            for (int r = 0; r < 3; ++r)
                for (int k = 0; k < 3; ++k) acc[3 * r + k] = add(acc[3 * r + k], mul(a[r], q[k]));
        } else {
            const double J[6] = {sub(mul(c[1], c[5]), mul(c[2], c[4])), sub(mul(c[2], c[3]), mul(c[0], c[5])),
                                 sub(mul(c[0], c[4]), mul(c[1], c[3])), c[3], c[4], c[5]};
            int k = 0;
            for (int r = 0; r < 6; ++r)
                for (int q = 0; q <= r; ++q, ++k) acc[k] = add(acc[k], mul(w, mul(J[r], J[q])));
            for (int r = 0; r < 6; ++r) acc[21 + r] = add(acc[21 + r], mul(-w, mul(J[r], c[6])));
        }
    }
    for (int k = 0; k < K; ++k) val[static_cast<size_t>(j) * K + k] = acc[k];
}

// the leaves pairwise up to the root (one block): level s adds leaf a + s into leaf a for a = 0, 2s, 4s, ...
template <int K>
__device__ void tree_sum(unsigned long long n, double* val) {
    const unsigned leaves = static_cast<unsigned>((n + kLeaf - 1) / kLeaf);
    for (unsigned s = 1; s < leaves; s <<= 1) {
        for (unsigned j = threadIdx.x; static_cast<unsigned long long>(j) * 2 * s < leaves; j += blockDim.x) {
            const unsigned a = j * 2 * s, b = a + s;
            if (b < leaves)
                for (int k = 0; k < K; ++k) val[static_cast<size_t>(a) * K + k] = add(val[static_cast<size_t>(a) * K + k], val[static_cast<size_t>(b) * K + k]);
        }
        __syncthreads();
    }
}

// point-to-point: weight sum and centroids (align_clouds.cpp:1644-1677)
__global__ void __launch_bounds__(kTreeThreads, 1) al_centroid_kernel(double* val, AlignState* st) {
    if (st->done) return;
    const unsigned long long n = st->n_pairs;
    if (n < kMinIcpPoints) {
        if (threadIdx.x == 0) st->done = 1;
        return;
    }
    tree_sum<7>(n, val);
    if (threadIdx.x != 0) return;
    st->solved_any = 1;
    const double wsum = val[0];
    if (!isfinite(wsum) || wsum <= 1e-12) {
        st->done = 1;
        return;
    }
    for (int d = 0; d < 3; ++d) {
        st->cx[d] = val[1 + d] / wsum;
        st->cq[d] = val[4 + d] / wsum;
    }
}

// point-to-point: covariance root, SVD, rotation, translation, composition and the stop test (:1679-1715)
__global__ void __launch_bounds__(kTreeThreads, 1) al_p2p_solve_kernel(double* val, AlignState* st) {
    if (st->done) return;
    tree_sum<9>(st->n_pairs, val);
    if (threadIdx.x != 0) return;
    st->iterations += 1;
    double u[3][3], v[3][3];
    bool ok = svd3(val, u, v);
    for (int i = 0; i < 3 && ok; ++i)
        for (int j = 0; j < 3; ++j) ok = ok && isfinite(u[i][j]) && isfinite(v[i][j]);
    if (!ok) {
        st->done = 1;
        return;
    }
    double R[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            R[3 * i + j] = add(add(mul(v[i][0], u[j][0]), mul(v[i][1], u[j][1])), mul(v[i][2], u[j][2]));
    const double det = add(sub(mul(R[0], sub(mul(R[4], R[8]), mul(R[5], R[7]))), mul(R[1], sub(mul(R[3], R[8]), mul(R[5], R[6])))),
                           mul(R[2], sub(mul(R[3], R[7]), mul(R[4], R[6]))));
    if (det < 0.0) {
        for (int i = 0; i < 3; ++i) v[i][2] = mul(v[i][2], -1.0);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                R[3 * i + j] = add(add(mul(v[i][0], u[j][0]), mul(v[i][1], u[j][1])), mul(v[i][2], u[j][2]));
    }
    double dt[3];
    for (int d = 0; d < 3; ++d)
        dt[d] = sub(st->cq[d], add(add(mul(R[3 * d], st->cx[0]), mul(R[3 * d + 1], st->cx[1])), mul(R[3 * d + 2], st->cx[2])));
    bool fin = finite3(dt);
    for (int i = 0; i < 9; ++i) fin = fin && isfinite(R[i]);
    if (!fin) {
        st->done = 1;
        return;
    }
    const double D[16] = {R[0], R[1], R[2], dt[0], R[3], R[4], R[5], dt[1], R[6], R[7], R[8], dt[2], 0.0, 0.0, 0.0, 1.0};
    pose_premul(D, st->pose);
    const double trace_term = smax(-1.0, smin(mul(0.5, sub(add(add(R[0], R[4]), R[8]), 1.0)), 1.0));
    if (acos(trace_term) < 1e-4 && norm3(dt) < 1e-3) st->done = 1;
}

// point-to-plane: the system's root, LDLT, PoseV::exp, composition and the stop test (:1816-1867)
__global__ void __launch_bounds__(kTreeThreads, 1) al_plane_solve_kernel(double* val, AlignState* st) {
    if (st->done) return;
    const unsigned long long n = st->n_pairs;
    if (n < kMinIcpPoints) {
        if (threadIdx.x == 0) st->done = 1;
        return;
    }
    tree_sum<27>(n, val);
    if (threadIdx.x != 0) return;
    st->solved_any = 1;
    st->iterations += 1;
    double H[36], b[6], dx[6];
    int k = 0;
    for (int r = 0; r < 6; ++r)
        for (int q = 0; q <= r; ++q, ++k) H[6 * r + q] = H[6 * q + r] = val[k];
    for (int r = 0; r < 6; ++r) {
        H[7 * r] = add(H[7 * r], 1e-10);
        b[r] = val[21 + r];
    }
    bool ok = ldlt_solve6(H, b, dx);
    for (int r = 0; r < 6; ++r) ok = ok && isfinite(dx[r]);
    if (!ok) {
        st->done = 1;
        return;
    }
    double E[16];
    posev_exp(dx, E);
    pose_premul(E, st->pose);
    if (norm3(dx) < 1e-4 && norm3(dx + 3) < 1e-3) st->done = 1;
}

__global__ void al_finish_kernel(const AlignState* st, double* pose, int32_t* iterations) {
    const double* src = st->solved_any ? st->pose : st->guess;
    for (int j = 0; j < 16; ++j) pose[j] = src[j];
    if (iterations) *iterations = st->iterations;
}

}  // namespace
}  // namespace ob

using namespace ob;

namespace {

size_t elem_size(int32_t dtype) { return dtype == OB_F64 ? 8 : 4; }

// SpatialHashGrid3D over `t` (with the normal filter when normals != null), built on the stream
template <typename T>
cudaError_t build_grid(const Rows& t, const void* normals, double cell_size, Staging& stg, cudaStream_t st, Grid* g) {
    const unsigned cap = std::max(t.cap, 1u);
    unsigned slots = 64;
    while (slots < 2 * cap) slots <<= 1;
    auto* keys = stg.scratch<GKey>(cap);
    auto* sk = stg.scratch<GKey>(cap);
    auto* seq = stg.scratch<uint32_t>(cap);
    auto* sseq = stg.scratch<uint32_t>(cap);
    auto* head = stg.scratch<uint32_t>(cap);
    auto* cid = stg.scratch<uint32_t>(cap);
    auto* cbeg = stg.scratch<uint32_t>(cap);
    auto* cend = stg.scratch<uint32_t>(cap);
    auto* row = stg.scratch<uint32_t>(cap);
    auto* ckey = stg.scratch<int64_t>(cap * 3ull);
    auto* pts = stg.scratch<double>(cap * 3ull);
    auto* table = stg.scratch<int32_t>(slots);
    const auto sort = sort_pairs(keys, sk, seq, sseq, static_cast<int>(cap), GKeyDecomposer{}, 0, kGKeyBits, st);
    const auto scan = inclusive_sum(head, cid, static_cast<int>(cap), st);
    CubTemp tmp(stg, sort, scan);
    cudaError_t e = stg.error();
    if (e == cudaSuccess) e = cudaMemsetAsync(table, 0xff, slots * 4ull, st);
    if (e != cudaSuccess) return e;
    const unsigned nb = blocks_for(cap);
    Rows tc = t;
    tc.cap = cap;  // rows_n() still clamps to the real count; rows past it get the pad bit
    if (t.cap == 0) tc.n_dev = nullptr, tc.n_host = 0;
    launch(OB_FAM_ALIGN, gr_key_kernel<T>, nb, 256, 0, st, tc, normals, 1.0 / cell_size, keys, seq);
    e = tmp.run(sort);
    if (e != cudaSuccess) return e;
    launch(OB_FAM_ALIGN, gr_head_kernel, nb, 256, 0, st, cap, sk, head);
    e = tmp.run(scan);
    if (e != cudaSuccess) return e;
    launch(OB_FAM_ALIGN, gr_fill_kernel<T>, nb, 256, 0, st, cap, t.p, sk, sseq, cid, ckey, cbeg, cend, table, slots - 1,
           pts, row);
    *g = Grid{ckey, cbeg, cend, table, slots - 1, pts, row, 1.0 / cell_size};
    return cudaGetLastError();
}

template <typename T>
ob_status run_align(const ob_cloud_align_io* io, const Rows& sr, const Rows& tr, const void* snrm, const void* tnrm,
                    const double* guess, Staging& stg, cudaStream_t st, double* pose, int32_t* iters) {
    const bool plane = io->mode == OB_ALIGN_POINT_TO_PLANE;
    Grid g{};
    cudaError_t e = build_grid<T>(tr, plane ? tnrm : nullptr, io->max_corr_dist, stg, st, &g);
    if (e != cudaSuccess) return fail_cuda(e, "cloud align grid");
    const unsigned kcap = std::max(sr.cap, 1u);
    const unsigned nb = (kcap + kThreads - 1) / kThreads;
    const unsigned slots = (kcap + kLeaf - 1) / kLeaf;
    auto* state = stg.scratch<AlignState>(1);
    auto* rows = stg.scratch<double>(static_cast<size_t>(kcap) * kPair);
    auto* pairs = stg.scratch<double>(static_cast<size_t>(kcap) * kPair);
    auto* val = stg.scratch<double>(slots * 27ull);
    auto* valid = stg.scratch<uint32_t>(kcap);
    auto* bc = stg.scratch<uint32_t>(nb);
    auto* keys = stg.scratch<unsigned long long>(kcap);
    auto* skeys = stg.scratch<unsigned long long>(kcap);
    const auto median_sort = sort_keys(keys, skeys, static_cast<int>(kcap), 0, 64, st);
    CubTemp tmp(stg, median_sort);
    e = stg.error();
    if (e != cudaSuccess) return fail_cuda(e, "cloud align workspace");
    const double max_d2 = io->max_corr_dist * io->max_corr_dist;
    const double cos_gate = plane ? std::cos(io->max_normal_angle_deg * M_PI / 180.0) : 0.0;
    const unsigned lb = (slots + 255) / 256;
    launch(OB_FAM_ALIGN, al_init_kernel, 1, 1, 0, st, sr, tr, guess, state);
    for (int it = 0; it < kMaxIterations; ++it) {
        if (plane)
            launch(OB_FAM_ALIGN, al_assoc_kernel<T, true>, nb, kThreads, 0, st, sr, snrm, tr.p, tnrm, g, max_d2,
                   cos_gate, kcap, state, rows, valid, bc, keys);
        else
            launch(OB_FAM_ALIGN, al_assoc_kernel<T, false>, nb, kThreads, 0, st, sr, nullptr, tr.p, nullptr, g, max_d2,
                   0.0, kcap, state, rows, valid, bc, keys);
        launch(OB_FAM_ALIGN, al_compact_kernel, nb, kThreads, 0, st, kcap, rows, valid, bc, pairs, state);
        e = tmp.run(median_sort);
        if (e != cudaSuccess) return fail_cuda(e, "cloud align median");
        if (plane) {
            launch(OB_FAM_ALIGN, al_leaf_kernel<kPlaneSystem>, lb, 256, 0, st, pairs, skeys, io->max_corr_dist, state,
                   slots, val);
            launch(OB_FAM_ALIGN, al_plane_solve_kernel, 1, kTreeThreads, 0, st, val, state);
        } else {
            launch(OB_FAM_ALIGN, al_leaf_kernel<kCentroid>, lb, 256, 0, st, pairs, skeys, io->max_corr_dist, state,
                   slots, val);
            launch(OB_FAM_ALIGN, al_centroid_kernel, 1, kTreeThreads, 0, st, val, state);
            launch(OB_FAM_ALIGN, al_leaf_kernel<kCovariance>, lb, 256, 0, st, pairs, skeys, io->max_corr_dist, state,
                   slots, val);
            launch(OB_FAM_ALIGN, al_p2p_solve_kernel, 1, kTreeThreads, 0, st, val, state);
        }
    }
    launch(OB_FAM_ALIGN, al_finish_kernel, 1, 1, 0, st, state, pose, iters);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "cloud align launch");
    return OB_OK;
}

}  // namespace

extern "C" {

ob_status ob_cloud_align(const ob_cloud_align_io* io, ob_stream* s) {
    if (!io || !s || !io->pose) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const bool plane = io->mode == OB_ALIGN_POINT_TO_PLANE;
    if (!plane && io->mode != OB_ALIGN_POINT_TO_POINT) return fail(OB_INVALID_ARGUMENT, "unknown align mode");
    // the reference's checks in its order (align_clouds.cpp:1593-1595, 1731-1747)
    if (!std::isfinite(io->max_corr_dist) || io->max_corr_dist <= 0.0)
        return fail(OB_INVALID_ARGUMENT, "max_corr_dist must be finite and greater than zero");
    const size_t src_rows = row_capacity(io->source.n, io->source.n_device, io->source.capacity);
    const size_t tgt_rows = row_capacity(io->target.n, io->target.n_device, io->target.capacity);
    if (plane) {
        if (!std::isfinite(io->max_normal_angle_deg) || io->max_normal_angle_deg < 0.0 || io->max_normal_angle_deg > 180.0)
            return fail(OB_INVALID_ARGUMENT, "max_normal_angle_deg must be finite and in [0, 180]");
        if (io->source_normal_rows != src_rows)
            return fail(OB_INVALID_ARGUMENT, "source_points and source_normals must have the same number of rows");
        if (io->target_normal_rows != tgt_rows)
            return fail(OB_INVALID_ARGUMENT, "target_points and target_normals must have the same number of rows");
        if ((src_rows && !io->source_normals) || (tgt_rows && !io->target_normals))
            return fail(OB_INVALID_ARGUMENT, "null normals buffer");
    }
    if (io->source.dtype != io->target.dtype) return fail(OB_INVALID_ARGUMENT, "source and target must share a dtype");
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    Rows sr{}, tr{};
    rs = stage_rows(&io->source, stg, &sr, "stage align source");
    if (rs == OB_OK) rs = stage_rows(&io->target, stg, &tr, "stage align target");
    if (rs != OB_OK) return rs;
    const size_t esz = elem_size(io->source.dtype);
    const void* snrm = plane ? stg.in(io->source_normals, sr.cap * 3 * esz) : nullptr;
    const void* tnrm = plane ? stg.in(io->target_normals, tr.cap * 3 * esz) : nullptr;
    const double* g = stg.in(io->initial_guess, 16);
    double* p = stg.out(io->pose, 16);
    int32_t* it = stg.out(io->iterations, 1);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage cloud align");
    rs = io->source.dtype == OB_F64 ? run_align<double>(io, sr, tr, snrm, tnrm, g, stg, st, p, it)
                                    : run_align<float>(io, sr, tr, snrm, tnrm, g, stg, st, p, it);
    if (rs != OB_OK) return rs;
    cudaError_t e = stg.finish();  // host pose / iterations: one wait; device ones: nothing waits for the GPU
    if (e != cudaSuccess) return fail_cuda(e, "cloud align result");
    return OB_OK;
}

ob_status ob_cloud_nearest(const ob_cloud_nearest_io* io, ob_stream* s) {
    if (!io || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (!std::isfinite(io->cell_size) || io->cell_size <= 0.0)
        return fail(OB_INVALID_ARGUMENT, "cell_size must be finite and greater than zero");
    if (io->target.dtype != io->queries.dtype) return fail(OB_INVALID_ARGUMENT, "target and queries must share a dtype");
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    Rows tr{}, qr{};
    rs = stage_rows(&io->target, stg, &tr, "stage nearest target");
    if (rs == OB_OK) rs = stage_rows(&io->queries, stg, &qr, "stage nearest queries");
    if (rs != OB_OK || qr.cap == 0) return rs;
    if (!io->indices) return fail(OB_INVALID_ARGUMENT, "null indices buffer");
    const void* nrm = stg.in(io->target_normals, tr.cap * 3 * elem_size(io->target.dtype));
    int32_t* out = stg.out(io->indices, qr.cap);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage nearest");
    Grid g{};
    cudaError_t e;
    if (io->target.dtype == OB_F64) {
        e = build_grid<double>(tr, nrm, io->cell_size, stg, st, &g);
        if (e == cudaSuccess)
            launch(OB_FAM_ALIGN, al_nearest_kernel<double>, blocks_for(qr.cap), 256, 0, st, qr, g, io->max_dist_sq,
                   out);
    } else {
        e = build_grid<float>(tr, nrm, io->cell_size, stg, st, &g);
        if (e == cudaSuccess)
            launch(OB_FAM_ALIGN, al_nearest_kernel<float>, blocks_for(qr.cap), 256, 0, st, qr, g, io->max_dist_sq,
                   out);
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    stg.check(e);
    e = stg.finish();
    if (e != cudaSuccess) return fail_cuda(e, "cloud nearest");
    return OB_OK;
}

}  // extern "C"
