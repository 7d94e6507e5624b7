// ob_ground.cu -- ground segmentation on the GPU (DESIGN f-13): the height-grid model of
// ouster_algorithm/src/ground_seg.cpp:666-1314 (build_lower_envelope_ground_model, xy_point_is_ground_like,
// get_ground_mask_into) for every frame of a set, each pass one launch over all frames.
//
// Every step is double arithmetic with one rounding per operation (explicit __dmul_rn / __dadd_rn, no contraction),
// and every statistic is a selection in the total order "<, then -0.0 before +0.0" (DESIGN §9), so each grid after
// each pass is bit-identical to oracle/orc_ground.c given the same normals.  Selections sort the order-preserving
// uint64 image of the double (okey()) as an unsigned key: CUB's floating-point radix digits fold -0.0 onto +0.0.
//
// Passes (launch family "ground"; CUB's own sort and scan kernels are not counted):
//   span         first / last column with status bit 0, per frame
//   points       dewarped model points (first two returns), extents (atomicMin/Max on okey()), z and footprint keys
//   [sort]       per frame: z and max(|x|, |y|) ascending
//   header       footprint bound, fallback z (sequential ascending sum, one thread per frame), origin, shape
//   -- the one host wait: grid shapes, then the grids are allocated --
//   cell keys    [sort by (cell, z)]  cell segments  [flag scan]  compact  cells
//   fill (6)  smooth  prune  fill (6)  smooth  components  fill (3)  -- Jacobi passes, one launch each (prune: one
//                                                                      CTA per frame, level-synchronous BFS)
//   classify     one thread per pixel per return
#include <algorithm>
#include <cmath>
#include <vector>

#include "ob_api_common.h"
#include "ob_arith.cuh"
#include "ob_cub.cuh"
#include "ob_project.cuh"

namespace ob {

namespace {

// constants of ground_seg.cpp:43-156 (as in oracle/orc_ground.c)
constexpr double kMinRange = 0.15, kNormalEps = 1e-6, kMadToSigma = 1.4826;
constexpr double kXyBoundsPct = 0.95, kIndoorBound = 25.0, kIndoorMaxZ = 0.3;
constexpr double kTailLow = 0.01, kTailHigh = 0.20;
constexpr double kCellLowPct = 0.15, kRoughBand = 0.45;
constexpr double kNzPrefilter = 0.15, kPointNzMin = 0.15, kWallNzMax = 0.45, kWallAboveLocal = 0.20;
constexpr unsigned kNfMinPoints = 4;
constexpr double kFillMaxSpread = 0.65, kSmoothMaxDiff = 0.55;
constexpr double kAnchorAbove = 1.10, kMaxNeighborStep = 0.75, kSlopePerM = 0.80, kPruneMinAbove = 1.50;
constexpr double kCompClose = 0.50, kCompHigh = 1.20, kCompModerateFrac = 0.20, kCompHighFrac = 0.80,
                 kCompMaxStep = 0.45;
constexpr int kLookupRadius = 8;
constexpr double kBaseTol = 0.50, kRoughK = 2.5, kNoiseK = 0.01, kNoiseMax = 0.50, kLookupTolPerM = 0.20,
                 kLookupTolMax = 0.45, kOutdoorMaxZ = 1.20, kMaxAboveLocal = 0.50, kMaxBelowLocal = 1.20,
                 kUnsupportedAbove = 0.90;
constexpr double kFloorPct = 0.05, kObstSpan = 0.55, kObstMinAbove = 0.25, kObstRoughCap = 0.10, kObstWallNz = 0.65,
                 kObstWallAbove = 0.20, kLiftMax = 0.25, kWallFloorHard = 0.35;
constexpr unsigned kObstMinPoints = 2;

constexpr int kThreads = 256;
constexpr int kFillWarps = 8;
constexpr unsigned long long kNoKey = ~0ull;

// one frame of the call, device memory
struct GFrame {
    const double* dir;    // h*w x 3, the item's f64 LUT
    const double* off;
    const uint32_t* range[2];  // model returns
    const uint32_t* const* ranges;  // every return (device table of n_ret pointers)
    uint8_t* const* masks;          // n_ret masks (device table), null entries skipped
    const uint32_t* status;
    const double* poses;
    const float* nrm[2];      // NORMALS / NORMALS2 or null
    const double* nrm64[2];   // normals computed by this call (ob_normals) or null
    // inputs of the computed normals, written by normals_input_kernel: dewarped points and range of the model
    // returns and the per-column sensor origins, each at the frame's place in its shape group's batch
    double* nxyz[2];
    uint32_t* nrange[2];
    double* norigin;
    const double* sensor_to_body;  // 16, row-major
    unsigned H, W, n_model, n_ret;
    unsigned long long pt_off;    // first point slot (n_model*H*W slots per frame)
    unsigned long long cell_off;  // first grid cell (after the host wait)
};

// per-frame state written by the kernels; the host reads it once (the grid shapes)
struct GState {
    int first, last;
    unsigned long long min_x, min_y, max_x, max_y;  // okey() images
    unsigned long long n_points;
    double origin_x, origin_y, fallback_z, footprint_bound, cell, inv;
    int rows, cols, valid, has_columns;
    int prune_levels, pad;
    unsigned long long best;  // main component: (size << 32) | ~local root
};

__device__ __forceinline__ void point_of(const GFrame& f, const uint32_t* range, unsigned row, unsigned col, double* p) {
    const size_t i = static_cast<size_t>(row) * f.W + col;
    const uint32_t r = range[i];
    const double q0 = project(r, f.dir[i * 3 + 0], f.off[i * 3 + 0]);
    const double q1 = project(r, f.dir[i * 3 + 1], f.off[i * 3 + 1]);
    const double q2 = project(r, f.dir[i * 3 + 2], f.off[i * 3 + 2]);
    const double* m = f.poses + static_cast<size_t>(col) * 16;
    p[0] = pose_row(m, q0, q1, q2);
    p[1] = pose_row(m + 4, q0, q1, q2);
    p[2] = pose_row(m + 8, q0, q1, q2);
}

// the frame's normal of return `ret` at pixel px, widened to double; false when the return has none
__device__ __forceinline__ bool normal_at(const GFrame& f, int ret, unsigned px, double& x, double& y, double& z) {
    if (ret < 0 || ret > 1) return false;
    if (f.nrm64[ret] != nullptr) {
        x = f.nrm64[ret][px * 3 + 0], y = f.nrm64[ret][px * 3 + 1], z = f.nrm64[ret][px * 3 + 2];
        return true;
    }
    if (f.nrm[ret] != nullptr) {
        x = f.nrm[ret][px * 3 + 0], y = f.nrm[ret][px * 3 + 1], z = f.nrm[ret][px * 3 + 2];
        return true;
    }
    return false;
}

// inputs of ob_normals for the frames whose normals this call computes (get_ground_mask_into, ground_seg.cpp:
// 1195-1250): every pixel's dewarped point (range 0 gives the column's translation, as cartesian then dewarp do),
// the range images, and the sensor origins (pose_c * sensor_to_body).translation summed ((a0 + a1) + a2) + a3
__global__ void normals_input_kernel(const GFrame* frames) {
    const GFrame& f = frames[blockIdx.y];
    if (f.norigin == nullptr) return;
    const unsigned hw = f.H * f.W;
    const unsigned long long n = static_cast<unsigned long long>(f.n_model) * hw + f.W;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        if (k < static_cast<unsigned long long>(f.n_model) * hw) {
            const unsigned ret = static_cast<unsigned>(k / hw), px = static_cast<unsigned>(k % hw);
            double p[3];
            point_of(f, f.range[ret], px / f.W, px % f.W, p);
            f.nxyz[ret][px * 3 + 0] = p[0];
            f.nxyz[ret][px * 3 + 1] = p[1];
            f.nxyz[ret][px * 3 + 2] = p[2];
            f.nrange[ret][px] = f.range[ret][px];
        } else {
            const unsigned col = static_cast<unsigned>(k - static_cast<unsigned long long>(f.n_model) * hw);
            const double* m = f.poses + static_cast<size_t>(col) * 16;
            const double* t = f.sensor_to_body;
            for (int i = 0; i < 3; ++i) {
                double acc = mul(m[i * 4 + 0], t[3]);
                acc = add(acc, mul(m[i * 4 + 1], t[7]));
                acc = add(acc, mul(m[i * 4 + 2], t[11]));
                acc = add(acc, mul(m[i * 4 + 3], t[15]));
                f.norigin[col * 3 + i] = acc;
            }
        }
    }
}

// ---- pass 1: column span, model points, extents ----
__global__ void span_kernel(const GFrame* frames, GState* gs) {
    const GFrame& f = frames[blockIdx.x];
    GState& s = gs[blockIdx.x];
    __shared__ int lo, hi;
    if (threadIdx.x == 0) lo = 0x7fffffff, hi = -1;
    __syncthreads();
    for (unsigned c = threadIdx.x; c < f.W; c += blockDim.x)
        if (f.status[c] & 1u) atomicMin(&lo, static_cast<int>(c)), atomicMax(&hi, static_cast<int>(c));
    __syncthreads();
    if (threadIdx.x == 0) {
        s.first = hi >= 0 ? lo : -1;
        s.last = hi;
        s.has_columns = hi >= 0;
        s.min_x = s.min_y = kNoKey;
        s.max_x = s.max_y = 0;
        s.n_points = 0;
        s.fallback_z = __longlong_as_double(0x7ff8000000000000ll);
        s.footprint_bound = 0.0;
        s.origin_x = s.origin_y = 0.0;
        s.rows = s.cols = s.valid = 0;
        s.prune_levels = 0;
        s.best = 0;
    }
}

// slot = ret*H*W + row*W + col.  keys: [0, P) z, [P, 2P) footprint; kNoKey for slots without a model point
__global__ void points_kernel(const GFrame* frames, GState* gs, double* pts, uint8_t* nflag,
                              unsigned long long* keys, uint32_t* groups, unsigned long long P, unsigned n_frames) {
    const unsigned fi = blockIdx.y;
    const GFrame& f = frames[fi];
    GState& s = gs[fi];
    const unsigned long long n = static_cast<unsigned long long>(f.n_model) * f.H * f.W;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long slot = f.pt_off + k;
        const unsigned hw = f.H * f.W;
        const unsigned ret = static_cast<unsigned>(k / hw), px = static_cast<unsigned>(k % hw);
        const unsigned row = px / f.W, col = px % f.W;
        unsigned long long zk = kNoKey, fk = kNoKey;
        uint8_t flag = 0;
        const int c = static_cast<int>(col);
        if (c >= s.first && c <= s.last && f.status[col] != 0u && f.range[ret][px] != 0u) {
            double p[3];
            point_of(f, f.range[ret], row, col, p);
            if (finite3(p[0], p[1], p[2]) && !(norm3(p[0], p[1], p[2]) < kMinRange)) {
                pts[slot * 3 + 0] = p[0];
                pts[slot * 3 + 1] = p[1];
                pts[slot * 3 + 2] = p[2];
                zk = okey(p[2]);
                fk = okey(fmax(fabs(p[0]), fabs(p[1])));
                atomicMin(&s.min_x, okey(p[0]));
                atomicMin(&s.min_y, okey(p[1]));
                atomicMax(&s.max_x, okey(p[0]));
                atomicMax(&s.max_y, okey(p[1]));
                atomicAdd(&s.n_points, 1ull);
                double x, y, z;
                if (normal_at(f, static_cast<int>(ret), px, x, y, z)) {
                    const double nn = norm3(x, y, z);
                    if (finite3(x, y, z) && nn > kNormalEps && fabs(z / nn) >= kNzPrefilter) flag = 1;
                }
            }
        }
        nflag[slot] = flag;
        keys[slot] = zk;
        keys[P + slot] = fk;
        groups[slot] = fi;
        groups[P + slot] = n_frames + fi;
    }
}

// ---- pass 2: footprint bound, fallback z, grid shape (one thread per frame) ----
// sorted: the keys grouped by frame (z groups, then footprint groups), ascending inside a group
__global__ void header_kernel(const GFrame* frames, GState* gs, const unsigned long long* sorted,
                              unsigned long long P, unsigned n_frames, double grid_size) {
    const unsigned fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= n_frames) return;
    const GFrame& f = frames[fi];
    GState& s = gs[fi];
    const unsigned long long n = s.n_points;
    if (n == 0) return;
    const unsigned long long* zs = sorted + f.pt_off;
    const unsigned long long* fp = sorted + P + f.pt_off;
    unsigned long long k = static_cast<unsigned long long>(floor(kXyBoundsPct * static_cast<double>(n - 1)));
    if (k > n - 1) k = n - 1;
    s.footprint_bound = okey_value(fp[k]);
    unsigned long long lo = static_cast<unsigned long long>(floor(kTailLow * static_cast<double>(n - 1)));
    unsigned long long hi = static_cast<unsigned long long>(ceil(kTailHigh * static_cast<double>(n - 1)));
    if (lo > n - 1) lo = n - 1;
    if (hi > n - 1) hi = n - 1;
    if (hi < lo) hi = lo;
    double sum = 0.0;
    for (unsigned long long i = lo; i <= hi; ++i) sum = add(sum, okey_value(zs[i]));  // ascending, as pinned in §9
    s.fallback_z = sum / static_cast<double>(hi - lo + 1);
    s.cell = grid_size;
    s.inv = 1.0 / grid_size;
    s.origin_x = mul(floor(mul(okey_value(s.min_x), s.inv)), s.cell);
    s.origin_y = mul(floor(mul(okey_value(s.min_y), s.inv)), s.cell);
    const double cols = ceil(sub(okey_value(s.max_x), s.origin_x) / s.cell) + 1.0;
    const double rows = ceil(sub(okey_value(s.max_y), s.origin_y) / s.cell) + 1.0;
    // the oracle's (int) conversion; a shape beyond int range is refused on the host
    s.cols = cols > 1.0 ? (cols < 2147483647.0 ? static_cast<int>(cols) : 0x7fffffff) : 1;
    s.rows = rows > 1.0 ? (rows < 2147483647.0 ? static_cast<int>(rows) : 0x7fffffff) : 1;
}

// ---- pass 3: cells ----
struct Grid {
    uint8_t* valid;
    uint8_t* obstacle;
    double* floor_z;
    double* height;
    double* rough;
};

__global__ void cell_keys_kernel(const GFrame* frames, const GState* gs, const double* pts,
                                 const unsigned long long* zkeys, uint32_t* ckeys, uint32_t* slots,
                                 uint32_t n_cells) {
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    const unsigned long long n = static_cast<unsigned long long>(f.n_model) * f.H * f.W;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long slot = f.pt_off + k;
        uint32_t key = n_cells;
        if (zkeys[slot] != kNoKey) {
            const int cc = static_cast<int>(floor(mul(sub(pts[slot * 3 + 0], s.origin_x), s.inv)));
            const int rr = static_cast<int>(floor(mul(sub(pts[slot * 3 + 1], s.origin_y), s.inv)));
            if (rr >= 0 && rr < s.rows && cc >= 0 && cc < s.cols)
                key = static_cast<uint32_t>(f.cell_off + static_cast<unsigned long long>(rr) * s.cols + cc);
        }
        ckeys[slot] = key;
        slots[slot] = static_cast<uint32_t>(slot);
    }
}

__global__ void gather_kernel(const uint32_t* src, const uint32_t* idx, uint32_t* out, unsigned long long n) {
    for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x)
        out[i] = src[idx[i]];
}

// sorted cell keys -> segment bounds; z and normal flags gathered in sorted order
__global__ void cell_segments_kernel(const uint32_t* skeys, const uint32_t* sslots, const unsigned long long* zkeys,
                                     const uint8_t* nflag, uint32_t* cbeg, uint32_t* cend, double* zs,
                                     uint32_t* flags, unsigned long long P, uint32_t n_cells) {
    for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < P;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const uint32_t key = skeys[i];
        uint32_t fl = 0;
        if (key < n_cells) {
            if (i == 0 || skeys[i - 1] != key) cbeg[key] = static_cast<uint32_t>(i);
            if (i + 1 == P || skeys[i + 1] != key) cend[key] = static_cast<uint32_t>(i + 1);
            const uint32_t slot = sslots[i];
            zs[i] = okey_value(zkeys[slot]);
            fl = nflag[slot];
        }
        flags[i] = fl;
    }
}

__global__ void compact_kernel(const uint32_t* flags, const uint32_t* scan, const double* zs, double* fz,
                               unsigned long long P) {
    for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < P;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x)
        if (flags[i]) fz[scan[i]] = zs[i];
}

// number of entries of sorted v[0, n) that are <= x, or < x (numeric comparisons)
__device__ __forceinline__ unsigned count_le(const double* v, unsigned n, double x) {
    unsigned lo = 0, hi = n;
    while (lo < hi) {
        const unsigned m = (lo + hi) >> 1;
        if (v[m] <= x) lo = m + 1; else hi = m;
    }
    return lo;
}
__device__ __forceinline__ unsigned count_lt(const double* v, unsigned n, double x) {
    unsigned lo = 0, hi = n;
    while (lo < hi) {
        const unsigned m = (lo + hi) >> 1;
        if (v[m] < x) lo = m + 1; else hi = m;
    }
    return lo;
}

// robust_spread of the band v[0, nb) (sorted) around h: the median of |v - h| is the (nb/2)-th smallest of two
// sorted runs -- |v - h| for v < h read leftwards from the split, and for v >= h read rightwards -- since one
// rounding is monotone.  Every |.| is >= +0, so the numeric order is the total order here.
__device__ double band_spread(const double* v, unsigned nb, double h) {
    if (nb < 2u) return 0.0;
    const unsigned s = count_lt(v, nb, h);
    const unsigned nl = s, nr = nb - s;
    const unsigned k = nb / 2u;
    auto L = [&](unsigned j) { return fabs(sub(v[s - 1 - j], h)); };
    auto R = [&](unsigned j) { return fabs(sub(v[s + j], h)); };
    unsigned lo = k + 1 > nr ? k + 1 - nr : 0u, hi = nl < k + 1 ? nl : k + 1;
    while (lo < hi) {  // the least i (taken from L) with L(i) >= R(k - i)
        const unsigned i = (lo + hi) >> 1, j = k + 1 - i;
        if (L(i) < R(j - 1)) lo = i + 1; else hi = i;
    }
    const unsigned i = lo, j = k + 1 - lo;
    double mad = -1.0;
    if (i > 0) mad = fmax(mad, L(i - 1));
    if (j > 0) mad = fmax(mad, R(j - 1));
    return isfinite(mad) ? mul(kMadToSigma, mad) : 0.0;
}

__global__ void cells_kernel(const GFrame* frames, GState* gs, const uint32_t* cbeg, const uint32_t* cend,
                             const double* zs, const uint32_t* scan, const double* fz, Grid g) {
    const GFrame& f = frames[blockIdx.y];
    GState& s = gs[blockIdx.y];
    const unsigned long long n = static_cast<unsigned long long>(s.rows) * s.cols;
    if (s.n_points == 0) return;
    const bool any_normals = f.nrm[0] || f.nrm[1] || f.nrm64[0] || f.nrm64[1];
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long ci = f.cell_off + k;
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        g.valid[ci] = 0;
        g.obstacle[ci] = 0;
        g.floor_z[ci] = nan;
        g.height[ci] = nan;
        g.rough[ci] = 0.0;
        const unsigned b = cbeg[ci], m = cend[ci] - b;
        if (m == 0) continue;
        const double* z = zs + b;
        const double z_max = z[m - 1];
        unsigned fi = static_cast<unsigned>(floor(kFloorPct * static_cast<double>(m - 1)));
        unsigned hi = static_cast<unsigned>(floor(kCellLowPct * static_cast<double>(m - 1)));
        if (fi > m - 1) fi = m - 1;
        if (hi > m - 1) hi = m - 1;
        const double floor_z = z[fi], h_all = z[hi];
        if (!isfinite(h_all) || !isfinite(floor_z)) continue;
        g.floor_z[ci] = floor_z;
        const unsigned above = m - count_le(z, m, add(floor_z, kObstMinAbove));
        const bool obstacle = sub(z_max, floor_z) > kObstSpan && above >= kObstMinPoints;
        if (obstacle) g.obstacle[ci] = 1;
        const double* fsel = fz + scan[b];
        const unsigned nf = scan[b + m] - scan[b];
        double h_f = nan;
        bool use_f = false;
        if (any_normals && nf >= kNfMinPoints) {
            unsigned idx = static_cast<unsigned>(floor(kCellLowPct * static_cast<double>(nf - 1)));
            if (idx > nf - 1) idx = nf - 1;
            h_f = fsel[idx];
            const bool lifted = isfinite(h_f) && h_f > add(h_all, kLiftMax);
            use_f = isfinite(h_f) && !lifted && !obstacle;
        }
        const double* sel = use_f ? fsel : z;
        const unsigned ns = use_f ? nf : m;
        const double h = obstacle ? floor_z : (use_f ? h_f : h_all);
        if (!isfinite(h) || ns == 0) continue;
        const unsigned nb = count_le(sel, ns, add(h, kRoughBand));
        double rough = band_spread(sel, nb, h);  // an empty band is {h}: spread 0
        if (obstacle) rough = fmin(rough, kObstRoughCap);
        g.valid[ci] = 1;
        g.height[ci] = h;
        g.rough[ci] = rough;
        s.valid = 1;
    }
}

// ---- pass 4: fills and smooths (Jacobi: read `in`, write `out`) ----
// k-th smallest (total order) of v[0, n) in shared memory, by rank counting across the warp
__device__ double warp_kth(const double* v, unsigned n, unsigned kk, double* slot, unsigned lane) {
    for (unsigned i = lane; i < n; i += 32) {
        const unsigned long long ki = okey(v[i]);
        unsigned less = 0, eq = 0;
        for (unsigned j = 0; j < n; ++j) {
            const unsigned long long kj = okey(v[j]);
            less += kj < ki;
            eq += kj == ki;
        }
        if (less <= kk && kk < less + eq) *slot = v[i];  // equal keys carry equal bits
    }
    __syncwarp();
    const double r = *slot;
    __syncwarp();
    return r;
}

template <int R>
__global__ void __launch_bounds__(kFillWarps * 32) fill_kernel(const GFrame* frames, const GState* gs, Grid in,
                                                               Grid out) {
    constexpr int D = 2 * R + 1, N = D * D;
    __shared__ double hs[kFillWarps][N], rs[kFillWarps][N], tmp[kFillWarps][N], res[kFillWarps];
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    const unsigned long long n = static_cast<unsigned long long>(s.rows) * s.cols;
    const int rows = s.rows, cols = s.cols;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(kFillWarps) + w; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * kFillWarps) {
        const unsigned long long ci = f.cell_off + k;
        uint8_t v = in.valid[ci];
        double h = in.height[ci], r = in.rough[ci];
        if (s.valid && !v) {
            const int cr = static_cast<int>(k / cols), cc = static_cast<int>(k % cols);
            unsigned cnt = 0;
            for (int base = 0; base < N; base += 32) {
                const int t = base + static_cast<int>(lane);
                bool ok = false;
                unsigned long long ni = 0;
                if (t < N) {
                    const int dr = t / D - R, dc = t % D - R;
                    const int rr = cr + dr, c2 = cc + dc;
                    if ((dr != 0 || dc != 0) && rr >= 0 && rr < rows && c2 >= 0 && c2 < cols) {
                        ni = f.cell_off + static_cast<unsigned long long>(rr) * cols + c2;
                        ok = in.valid[ni] && isfinite(in.height[ni]);
                    }
                }
                const unsigned m = __ballot_sync(0xffffffffu, ok);
                if (ok) {
                    const unsigned pos = cnt + __popc(m & ((1u << lane) - 1u));
                    hs[w][pos] = in.height[ni];
                    rs[w][pos] = in.rough[ni];
                }
                cnt += __popc(m);
            }
            __syncwarp();
            if (cnt > 0) {  // the cheap rejection: no valid neighbour within the radius
                const double fill_h = warp_kth(hs[w], cnt, cnt / 2u, &res[w], lane);
                double spread = 0.0;
                if (cnt >= 2u && isfinite(fill_h)) {
                    for (unsigned i = lane; i < cnt; i += 32) tmp[w][i] = fabs(sub(hs[w][i], fill_h));
                    __syncwarp();
                    const double mad = warp_kth(tmp[w], cnt, cnt / 2u, &res[w], lane);
                    spread = isfinite(mad) ? mul(kMadToSigma, mad) : 0.0;
                }
                const double fill_r = warp_kth(rs[w], cnt, cnt / 2u, &res[w], lane);
                if (isfinite(fill_h) && !(spread > kFillMaxSpread)) {
                    v = 1;
                    h = fill_h;
                    r = fill_r;
                }
            }
        }
        if (lane == 0) {
            out.valid[ci] = v;
            out.height[ci] = h;
            out.rough[ci] = r;
        }
        __syncwarp();
    }
}

__device__ __forceinline__ double small_median(double* v, unsigned n) {  // insertion sort in the total order
    for (unsigned i = 1; i < n; ++i) {
        const double x = v[i];
        const unsigned long long kx = okey(x);
        unsigned j = i;
        while (j > 0 && okey(v[j - 1]) > kx) {
            v[j] = v[j - 1];
            --j;
        }
        v[j] = x;
    }
    return v[n / 2u];
}

__global__ void smooth_kernel(const GFrame* frames, const GState* gs, Grid in, Grid out) {
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    const unsigned long long n = static_cast<unsigned long long>(s.rows) * s.cols;
    const int rows = s.rows, cols = s.cols;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long ci = f.cell_off + k;
        const uint8_t v = in.valid[ci];
        double h = in.height[ci], r = in.rough[ci];
        if (s.valid && v && isfinite(h)) {
            const int cr = static_cast<int>(k / cols), cc = static_cast<int>(k % cols);
            double hs[9], rs[9];
            unsigned cnt = 0;
            for (int dr = -1; dr <= 1; ++dr)
                for (int dc = -1; dc <= 1; ++dc) {
                    const int rr = cr + dr, c2 = cc + dc;
                    if (rr < 0 || rr >= rows || c2 < 0 || c2 >= cols) continue;
                    const unsigned long long ni = f.cell_off + static_cast<unsigned long long>(rr) * cols + c2;
                    const double nh = in.height[ni];
                    if (!in.valid[ni] || !isfinite(nh)) continue;
                    if (fabs(sub(nh, in.height[ci])) > kSmoothMaxDiff) continue;
                    hs[cnt] = nh;
                    rs[cnt] = in.rough[ni];
                    ++cnt;
                }
            if (cnt) {
                h = small_median(hs, cnt);
                r = small_median(rs, cnt);
            }
        }
        out.valid[ci] = v;
        out.height[ci] = h;
        out.rough[ci] = r;
    }
}

// ---- pass 5: prune (one CTA per frame; level-synchronous BFS over one worklist, in place) ----
__global__ void __launch_bounds__(1024) prune_kernel(const GFrame* frames, GState* gs, Grid g, uint32_t* reach,
                                                     uint32_t* queue) {
    const GFrame& f = frames[blockIdx.x];
    GState& s = gs[blockIdx.x];
    if (!s.valid || !isfinite(s.fallback_z)) return;
    const unsigned n = static_cast<unsigned>(static_cast<unsigned long long>(s.rows) * s.cols);
    const int rows = s.rows, cols = s.cols;
    uint8_t* valid = g.valid + f.cell_off;
    double* height = g.height + f.cell_off;
    const uint8_t* obstacle = g.obstacle + f.cell_off;
    uint32_t* rc = reach + f.cell_off;
    uint32_t* q = queue + f.cell_off;
    __shared__ unsigned tail, levels;
    if (threadIdx.x == 0) tail = 0, levels = 0;
    __syncthreads();
    const double anchor = add(s.fallback_z, kAnchorAbove);
    for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
        rc[i] = 0;
        if (valid[i] && isfinite(height[i]) && height[i] <= anchor) {
            rc[i] = 1;
            q[atomicAdd(&tail, 1u)] = i;
        }
    }
    __syncthreads();
    if (tail == 0) return;
    const int DR[8] = {-1, -1, -1, 0, 0, 1, 1, 1}, DC[8] = {-1, 0, 1, -1, 1, -1, 0, 1};
    const double straight = add(0.25, mul(kSlopePerM, mul(s.cell, sqrt(1.0))));
    const double diagonal = add(0.25, mul(kSlopePerM, mul(s.cell, sqrt(2.0))));
    const double allowed_s = fmin(kMaxNeighborStep, straight), allowed_d = fmin(kMaxNeighborStep, diagonal);
    unsigned head = 0;
    while (true) {
        const unsigned end = tail;
        __syncthreads();
        if (head == end) break;
        for (unsigned e = head + threadIdx.x; e < end; e += blockDim.x) {
            const unsigned idx = q[e];
            const int r = static_cast<int>(idx / cols), c = static_cast<int>(idx % cols);
            const double h = height[idx];
            for (int d = 0; d < 8; ++d) {
                const int rr = r + DR[d], cc = c + DC[d];
                if (rr < 0 || rr >= rows || cc < 0 || cc >= cols) continue;
                const unsigned ni = static_cast<unsigned>(rr) * cols + cc;
                if (*(volatile uint32_t*)&rc[ni] || !valid[ni] || !isfinite(height[ni])) continue;
                const double allowed = (DR[d] != 0 && DC[d] != 0) ? allowed_d : allowed_s;
                if (fabs(sub(height[ni], h)) > allowed) continue;
                if (sub(height[ni], h) > 0.50 && obstacle[ni]) continue;
                if (atomicExch(&rc[ni], 1u) == 0u) q[atomicAdd(&tail, 1u)] = ni;
            }
        }
        head = end;
        if (threadIdx.x == 0) ++levels;
        __syncthreads();
    }
    const double cut = add(s.fallback_z, kPruneMinAbove);
    for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
        if (!valid[i] || !isfinite(height[i])) continue;
        if (!rc[i] && height[i] > cut) {
            valid[i] = 0;
            height[i] = __longlong_as_double(0x7ff8000000000000ll);
            g.rough[f.cell_off + i] = 0.0;
        }
    }
    if (threadIdx.x == 0) s.prune_levels = static_cast<int>(levels);
}

// ---- pass 6: components (union-find hooking the larger root under the smaller: root = lowest cell) ----
__device__ __forceinline__ bool comp_cell(const Grid& g, unsigned long long ci) {
    return g.valid[ci] && isfinite(g.height[ci]);
}

// find with path halving (ECL-CC): a cell's parent only ever moves to a lower ancestor, so every write keeps it in
// its set and roots stay the lowest cells
__device__ __forceinline__ uint32_t find_root(uint32_t* parent, uint32_t x) {
    volatile uint32_t* vp = parent;
    uint32_t p = vp[x];
    while (p != x) {
        const uint32_t gp = vp[p];
        if (gp != p) vp[x] = gp;
        x = p;
        p = vp[x];
    }
    return x;
}

__global__ void comp_init_kernel(const GFrame* frames, const GState* gs, uint32_t* parent, uint32_t* csize) {
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    const unsigned long long n = static_cast<unsigned long long>(s.rows) * s.cols;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        parent[f.cell_off + k] = static_cast<uint32_t>(f.cell_off + k);
        csize[f.cell_off + k] = 0;
    }
}

__global__ void comp_hook_kernel(const GFrame* frames, const GState* gs, Grid g, uint32_t* parent) {
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    if (!s.valid || !isfinite(s.fallback_z)) return;
    const unsigned long long n = static_cast<unsigned long long>(s.rows) * s.cols;
    const int rows = s.rows, cols = s.cols;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long ci = f.cell_off + k;
        if (!comp_cell(g, ci)) continue;
        const int r = static_cast<int>(k / cols), c = static_cast<int>(k % cols);
        const int DR[4] = {0, 1, 1, 1}, DC[4] = {1, -1, 0, 1};  // the edge is symmetric: half the 8 neighbours
        for (int d = 0; d < 4; ++d) {
            const int rr = r + DR[d], cc = c + DC[d];
            if (rr < 0 || rr >= rows || cc < 0 || cc >= cols) continue;
            const unsigned long long ni = f.cell_off + static_cast<unsigned long long>(rr) * cols + cc;
            if (!comp_cell(g, ni) || fabs(sub(g.height[ni], g.height[ci])) > kCompMaxStep) continue;
            uint32_t a = static_cast<uint32_t>(ci), b = static_cast<uint32_t>(ni);
            while (true) {
                a = find_root(parent, a);
                b = find_root(parent, b);
                if (a == b) break;
                if (a < b) { const uint32_t t = a; a = b; b = t; }  // a: the larger root, hooked under b
                if (atomicCAS(&parent[a], a, b) == a) break;
            }
        }
    }
}

// roots, component sizes and the (height, root) sort keys; cells outside every component get kNoKey / n_cells
__global__ void comp_roots_kernel(const GFrame* frames, const GState* gs, Grid g, uint32_t* parent, uint32_t* csize,
                                  unsigned long long* hkeys, uint32_t* cells, uint32_t n_cells) {
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    const unsigned long long n = static_cast<unsigned long long>(s.rows) * s.cols;
    const bool on = s.valid && isfinite(s.fallback_z);
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long ci = f.cell_off + k;
        unsigned long long hk = kNoKey;
        if (on && comp_cell(g, ci)) {
            const uint32_t root = find_root(parent, static_cast<uint32_t>(ci));
            parent[ci] = root;
            atomicAdd(&csize[root], 1u);
            hk = okey(g.height[ci]);
        }
        hkeys[ci] = hk;
        cells[ci] = static_cast<uint32_t>(ci);
    }
}

// after the (root, height) sort: each component's median height, and the main component per frame
__global__ void comp_median_kernel(const GFrame* frames, GState* gs, const uint32_t* sroot, const uint32_t* scell,
                                   const uint32_t* csize, const Grid g, double* med, unsigned n_frames,
                                   uint32_t n_cells) {
    for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n_cells;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const uint32_t r = sroot[i];
        if (r >= n_cells || (i > 0 && sroot[i - 1] == r)) continue;
        const uint32_t k = csize[r];
        const double m = g.height[scell[i + k / 2u]];
        med[r] = m;
        unsigned lo = 0, hi = n_frames;  // the frame of cell r: the last with cell_off <= r
        while (hi - lo > 1) {
            const unsigned mid = (lo + hi) >> 1;
            if (frames[mid].cell_off <= r) lo = mid; else hi = mid;
        }
        GState& s = gs[lo];
        if (isfinite(m) && m <= add(s.fallback_z, kAnchorAbove)) {
            const uint32_t local = static_cast<uint32_t>(r - frames[lo].cell_off);
            atomicMax(&s.best, (static_cast<unsigned long long>(k) << 32) | (0xffffffffu - local));
        }
    }
}

__global__ void comp_reject_kernel(const GFrame* frames, const GState* gs, Grid g, const uint32_t* parent,
                                   const uint32_t* csize, const double* med) {
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    if (!s.valid || !isfinite(s.fallback_z) || s.best == 0) return;
    const unsigned long long n = static_cast<unsigned long long>(s.rows) * s.cols;
    const unsigned long long main_root = f.cell_off + (0xffffffffu - static_cast<uint32_t>(s.best & 0xffffffffu));
    const double main_med = med[main_root];
    const double main_size = static_cast<double>(s.best >> 32);
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long ci = f.cell_off + k;
        if (!comp_cell(g, ci)) continue;
        const uint32_t r = parent[ci];
        if (r == main_root || !isfinite(med[r])) continue;
        const double dz = sub(med[r], main_med);
        const double frac = static_cast<double>(csize[r]) / main_size;
        if (fabs(dz) <= kCompClose) continue;
        if (dz > kCompClose && dz <= kCompHigh && frac >= kCompModerateFrac) continue;
        if (dz > kCompHigh && frac >= kCompHighFrac) continue;
        if (dz < -kCompClose && dz >= -kCompHigh) continue;
        g.valid[ci] = 0;
        g.height[ci] = __longlong_as_double(0x7ff8000000000000ll);
        g.rough[ci] = 0.0;
    }
}

// ---- pass 7: classification (xy_point_is_ground_like, ground_seg.cpp:947-1088) ----
__device__ __forceinline__ double abs_normal_z(const GFrame& f, int ret, unsigned px) {
    double x, y, z;
    if (!normal_at(f, ret, px, x, y, z)) return __longlong_as_double(0x7ff8000000000000ll);
    if (!finite3(x, y, z)) return __longlong_as_double(0x7ff8000000000000ll);
    const double nn = norm3(x, y, z);
    if (nn <= kNormalEps) return __longlong_as_double(0x7ff8000000000000ll);
    return fabs(z / nn);
}

__device__ bool ground_like(const GState& s, const GFrame& f, const Grid& g, const double* p, double range,
                            double fallback, int ret, unsigned px) {
    const bool has_normals = ret >= 0 && ret < 2 && (f.nrm[ret] != nullptr || f.nrm64[ret] != nullptr);
    const int rows = s.rows, cols = s.cols;
    const bool indoor = s.footprint_bound <= kIndoorBound;
    const double eff = isfinite(s.fallback_z) ? s.fallback_z : fallback;
    if (indoor && isfinite(eff) && p[2] > add(eff, kIndoorMaxZ)) return false;
    bool in_grid = false;
    int cr = 0, cc = 0;
    if (s.valid && finite3(p[0], p[1], p[2])) {
        cc = static_cast<int>(floor(mul(sub(p[0], s.origin_x), s.inv)));
        cr = static_cast<int>(floor(mul(sub(p[1], s.origin_y), s.inv)));
        in_grid = cr >= 0 && cr < rows && cc >= 0 && cc < cols;
    }
    if (in_grid) {
        const unsigned long long ci = f.cell_off + static_cast<unsigned long long>(cr) * cols + cc;
        if (g.obstacle[ci] && isfinite(g.floor_z[ci])) {
            const double above = sub(p[2], g.floor_z[ci]);
            if (above > kWallFloorHard) return false;
            const double nz = abs_normal_z(f, ret, px);
            if (isfinite(nz) && nz < kObstWallNz && above > kObstWallAbove) return false;
        }
        double lh = 0.0, lr = 0.0, ld = 0.0;
        bool found = false;
        if (g.valid[ci] && isfinite(g.height[ci])) {
            lh = g.height[ci];
            lr = g.rough[ci];
            found = true;
        } else {
            int best = 0x7fffffff;
            unsigned long long bi = 0;
            for (int rad = 1; rad <= kLookupRadius && !found; ++rad) {
                for (int dr = -rad; dr <= rad; ++dr)
                    for (int dc = -rad; dc <= rad; ++dc) {
                        if (max(abs(dr), abs(dc)) != rad) continue;
                        const int rr = cr + dr, c2 = cc + dc;
                        if (rr < 0 || rr >= rows || c2 < 0 || c2 >= cols) continue;
                        const unsigned long long ni = f.cell_off + static_cast<unsigned long long>(rr) * cols + c2;
                        if (!g.valid[ni] || !isfinite(g.height[ni])) continue;
                        const int d2 = dr * dr + dc * dc;
                        if (d2 < best) {
                            best = d2;
                            bi = ni;
                            found = true;
                        }
                    }
                if (found) {
                    lh = g.height[bi];
                    lr = g.rough[bi];
                    ld = mul(sqrt(static_cast<double>(best)), s.cell);
                }
            }
        }
        if (found) {
            const double fr = isfinite(lr) ? fmax(0.0, lr) : 0.0;
            const double noise = isfinite(range) ? fmin(kNoiseMax, mul(kNoiseK, fmax(0.0, range))) : kNoiseMax;
            const double extra = isfinite(ld) ? fmin(kLookupTolMax, mul(kLookupTolPerM, fmax(0.0, ld))) : 0.0;
            double tol = add(add(add(kBaseTol, mul(kRoughK, fr)), noise), extra);
            tol = fmin(tol, kMaxAboveLocal);
            if (indoor) tol = fmin(tol, kIndoorMaxZ);
            const double res = sub(p[2], lh);
            const double nz = abs_normal_z(f, ret, px);
            if (has_normals && res > kWallAboveLocal && isfinite(nz) && nz < kWallNzMax) return false;
            if (res > 0.35 && isfinite(nz) && nz < kPointNzMin) return false;
            return res <= tol && res >= -kMaxBelowLocal;
        }
    }
    if (s.valid) {
        if (!isfinite(eff)) return false;
        const double res = sub(p[2], eff);
        const double nz = abs_normal_z(f, ret, px);
        if (res > 0.35 && isfinite(nz) && nz < kPointNzMin) return false;
        const double cap = indoor ? kIndoorMaxZ : kUnsupportedAbove;
        return res <= cap && res >= -kMaxBelowLocal;
    }
    if (!isfinite(eff)) return false;
    return p[2] <= add(eff, indoor ? kIndoorMaxZ : kOutdoorMaxZ);
}

// classify = 0: masks are only zeroed (a call that stops before the last pass)
__global__ void classify_kernel(const GFrame* frames, const GState* gs, Grid g, int classify) {
    const GFrame& f = frames[blockIdx.y];
    const GState& s = gs[blockIdx.y];
    const unsigned hw = f.H * f.W;
    const unsigned long long n = static_cast<unsigned long long>(f.n_ret) * hw;
    const double fallback = isfinite(s.fallback_z) ? s.fallback_z : 0.0;
    for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
         k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned ret = static_cast<unsigned>(k / hw), px = static_cast<unsigned>(k % hw);
        uint8_t* mask = f.masks[ret];
        if (mask == nullptr) continue;
        const unsigned row = px / f.W, col = px % f.W;
        uint8_t out = 0;
        const int c = static_cast<int>(col);
        const uint32_t* range = f.ranges[ret];
        if (classify && s.first >= 0 && c >= s.first && c <= s.last && f.status[col] != 0u && range[px] != 0u) {
            double p[3];
            point_of(f, range, row, col, p);
            if (finite3(p[0], p[1], p[2])) {
                out = ground_like(s, f, g, p, norm3(p[0], p[1], p[2]), fallback, static_cast<int>(ret), px) ? 1 : 0;
            }
        }
        mask[px] = out;
    }
}

// the model header of every frame that asks for it (device scratch, staged to the caller's pointer)
__global__ void model_kernel(const GState* gs, ob_ground_model* out, unsigned n_frames) {
    const unsigned fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= n_frames) return;
    const GState& s = gs[fi];
    ob_ground_model m;
    m.origin_x = s.origin_x;
    m.origin_y = s.origin_y;
    m.fallback_z = s.fallback_z;
    m.footprint_bound = s.footprint_bound;
    m.rows = s.rows;
    m.cols = s.cols;
    m.valid = s.valid;
    m.has_columns = s.has_columns;
    out[fi] = m;
}

unsigned blocks_for(unsigned long long n, unsigned threads) {
    const unsigned long long b = (n + threads - 1) / threads;
    return static_cast<unsigned>(std::max<unsigned long long>(1, std::min<unsigned long long>(b, 1u << 16)));
}

// the root of each height-sorted cell (n_cells for cells outside every component), for the stable sort by root
__global__ void root_keys_kernel(const unsigned long long* hk_sorted, const uint32_t* cells, const uint32_t* parent,
                                 uint32_t* roots, unsigned long long n, uint32_t n_cells) {
    for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x)
        roots[i] = hk_sorted[i] == kNoKey ? n_cells : parent[cells[i]];
}

}  // namespace

}  // namespace ob

using namespace ob;

extern "C" ob_status ob_ground_mask(const ob_ground_item* items, size_t n_items, double grid_size, int stop,
                                    ob_stream* s) {
    if (n_items && !items) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (!(grid_size > 0.0) || !std::isfinite(grid_size))
        return fail(OB_INVALID_ARGUMENT, "GroundSegConfig.grid_size must be > 0");
    if (stop < 0 || stop > OB_GROUND_FINAL) return fail(OB_INVALID_ARGUMENT, "ground: stop must be in [0, OB_GROUND_FINAL]");
    for (size_t i = 0; i < n_items; ++i) {
        const ob_ground_item& it = items[i];
        if (!it.lut) continue;
        if (it.n_returns == 0 || !it.range || !it.range[0])
            return fail(OB_INVALID_ARGUMENT, "frame must contain RANGE field for get_ground_mask");
        for (size_t r = 1; r < it.n_returns; ++r)
            if (!it.range[r]) return fail(OB_INVALID_ARGUMENT, "frame must contain RANGE field for get_ground_mask");
        if (it.n_masks < it.n_returns || (it.n_returns && !it.masks))
            return fail(OB_INVALID_ARGUMENT, "not enough output masks provided for get_ground_mask_into");
        if (it.mask_h != it.h || it.mask_w != it.w)
            return fail(OB_INVALID_ARGUMENT, "output mask shape does not match frame shape");
        if (it.w && (!it.status || !it.poses)) return fail(OB_INVALID_ARGUMENT, "null pointer");
        if (it.compute_normals && !it.normals && !it.sensor_to_body) return fail(OB_INVALID_ARGUMENT, "null pointer");
        if (it.h * it.w > (1ull << 28)) return fail(OB_INVALID_ARGUMENT, "frame too large");
    }
    if (!s) {
        ob_status rs = require_device(0);
        return rs != OB_OK ? rs : fail(OB_INVALID_ARGUMENT, "null pointer");
    }
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    for (size_t i = 0; i < n_items; ++i) {
        if (!items[i].lut || items[i].h * items[i].w == 0) continue;  // no pixel: nothing to read or write
        const LutView lv = lut_view(items[i].lut);
        if (lv.dtype != OB_F64) return fail(OB_INVALID_ARGUMENT, "ground segmentation needs a float64 lut");
        if (lv.h != items[i].h || lv.w != items[i].w)
            return fail(OB_INVALID_ARGUMENT, "lut shape does not match frame shape");
    }
    const cudaStream_t st = stream_handle(s);
    Staging stg(st);
    std::vector<GFrame> frames;
    std::vector<size_t> slot_of;
    std::vector<const uint32_t*> rtab;
    std::vector<uint8_t*> mtab;
    std::vector<size_t> rbase;
    unsigned long long P = 0;
    unsigned max_slots = 0, max_px = 0;
    for (size_t i = 0; i < n_items && !stg.error(); ++i) {
        const ob_ground_item& it = items[i];
        if (!it.lut || it.h * it.w == 0) continue;
        const LutView lv = lut_view(it.lut);
        GFrame f{};
        const size_t npx = it.h * it.w;
        f.dir = static_cast<const double*>(lv.dir);
        f.off = static_cast<const double*>(lv.off);
        f.H = static_cast<unsigned>(it.h);
        f.W = static_cast<unsigned>(it.w);
        f.n_ret = static_cast<unsigned>(it.n_returns);
        f.n_model = it.n_returns >= 2 ? 2 : 1;
        rbase.push_back(rtab.size());
        for (size_t r = 0; r < it.n_returns; ++r) {
            rtab.push_back(stg.in(it.range[r], npx));
            mtab.push_back(stg.out(it.masks[r], npx));
        }
        for (unsigned r = 0; r < f.n_model; ++r) f.range[r] = rtab[rbase.back() + r];
        f.status = stg.in(it.status, it.w);
        f.poses = stg.in(it.poses, it.w * 16);
        // NORMALS2 is read only alongside NORMALS, and only for a second return
        if (it.normals) f.nrm[0] = stg.in(it.normals, npx * 3);
        if (it.normals && it.normals2 && f.n_model == 2) f.nrm[1] = stg.in(it.normals2, npx * 3);
        if (it.compute_normals && !it.normals) f.sensor_to_body = stg.in(it.sensor_to_body, 16);
        f.pt_off = P;
        P += static_cast<unsigned long long>(f.n_model) * npx;
        max_slots = std::max<unsigned>(max_slots, static_cast<unsigned>(f.n_model * npx));
        max_px = std::max<unsigned>(max_px, static_cast<unsigned>(it.n_returns * npx));
        frames.push_back(f);
        slot_of.push_back(i);
    }
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage ground buffers");
    const unsigned F = static_cast<unsigned>(frames.size());
    if (F == 0) return OB_OK;
    if (F > 65535) return fail(OB_INVALID_ARGUMENT, "too many frames in one call");
    if (P >= 0xffffffffull) return fail(OB_INVALID_ARGUMENT, "frame set too large");
    // the device tables of range and mask pointers
    const uint32_t* const* drt = stg.in(rtab.data(), rtab.size());
    uint8_t* const* dmt = stg.in(mtab.data(), mtab.size());
    for (unsigned k = 0; k < F; ++k) {
        frames[k].ranges = drt + rbase[k];
        frames[k].masks = dmt + rbase[k];
    }
    const unsigned long long P2 = 2 * P;
    auto* df = stg.scratch<GFrame>(F);
    auto* gs = stg.scratch<GState>(F);
    auto* pts = stg.scratch<double>(P * 3);
    auto* nflag = stg.scratch<uint8_t>(P);
    auto* k1 = stg.scratch<unsigned long long>(P2);
    auto* k2 = stg.scratch<unsigned long long>(P2);
    auto* k3 = stg.scratch<unsigned long long>(P2);
    auto* u1 = stg.scratch<uint32_t>(P2);
    auto* u2 = stg.scratch<uint32_t>(P2);
    // computed normals: frames of one shape and return count form one batch of ob_normals
    struct NormalsBatch {
        unsigned H, W, n_model;
        std::vector<unsigned> frames;
        double *xyz[2], *out[2], *origins, *subtent;
        uint32_t* range[2];
    };
    std::vector<NormalsBatch> batches;
    std::vector<int> batch_of(F, -1), index_in_batch(F, 0);
    unsigned max_norm = 0;
    for (unsigned k = 0; k < F; ++k) {
        if (!frames[k].sensor_to_body) continue;
        int b = -1;
        for (size_t j = 0; j < batches.size(); ++j)
            if (batches[j].H == frames[k].H && batches[j].W == frames[k].W && batches[j].n_model == frames[k].n_model)
                b = static_cast<int>(j);
        if (b < 0) {
            batches.push_back(NormalsBatch{frames[k].H, frames[k].W, frames[k].n_model, {}, {}, {}, nullptr, nullptr, {}});
            b = static_cast<int>(batches.size()) - 1;
        }
        batch_of[k] = b;
        index_in_batch[k] = static_cast<int>(batches[b].frames.size());
        batches[b].frames.push_back(k);
        max_norm = std::max(max_norm, frames[k].n_model * frames[k].H * frames[k].W + frames[k].W);
    }
    for (NormalsBatch& b : batches) {
        const size_t nb = b.frames.size(), hw = static_cast<size_t>(b.H) * b.W;
        for (unsigned r = 0; r < b.n_model; ++r) {
            b.xyz[r] = stg.scratch<double>(nb * hw * 3);
            b.out[r] = stg.scratch<double>(nb * hw * 3);
            b.range[r] = stg.scratch<uint32_t>(nb * hw);
        }
        b.origins = stg.scratch<double>(nb * b.W * 3);
        b.subtent = stg.scratch<double>(nb);
        if (stg.error()) break;
        for (size_t j = 0; j < nb; ++j) {
            GFrame& f = frames[b.frames[j]];
            for (unsigned r = 0; r < b.n_model; ++r) {
                f.nxyz[r] = b.xyz[r] + j * hw * 3;
                f.nrange[r] = b.range[r] + j * hw;
                f.nrm64[r] = b.out[r] + j * hw * 3;
            }
            f.norigin = b.origins + j * b.W * 3;
        }
    }
    cudaError_t e = stg.error();
    if (e == cudaSuccess) e = cudaMemcpyAsync(df, frames.data(), F * sizeof(GFrame), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return fail_cuda(e, "stage ground buffers");
    if (!batches.empty()) {
        launch(OB_FAM_GROUND, normals_input_kernel, dim3(blocks_for(max_norm, kThreads), F), kThreads, 0, st, df);
        e = cudaGetLastError();
        if (e != cudaSuccess) return fail_cuda(e, "ground normals");
        for (const NormalsBatch& b : batches) {  // the reference's normals() defaults (normals.h:23-25)
            ob_normals_io io{};
            io.n_frames = b.frames.size();
            io.h = b.H;
            io.w = b.W;
            io.xyz = b.xyz[0];
            io.range = b.range[0];
            io.normals = b.out[0];
            if (b.n_model == 2) io.xyz2 = b.xyz[1], io.range2 = b.range[1], io.normals2 = b.out[1];
            io.sensor_origins_xyz = b.origins;
            io.n_origins = b.W;
            io.origins_frame_stride = static_cast<size_t>(b.W) * 3;
            io.pixel_search_range = 1;
            io.min_angle_of_incidence_rad = 1.0 * M_PI / 180.0;
            io.target_distance_m = 0.025;
            io.vertical_subtent_out = b.subtent;
            const ob_status ns = ob_normals(OB_F64, &io, s);
            if (ns != OB_OK) return ns;
        }
    }

    // pass 1 and 2: points, extents, the per-frame sorts, the header
    launch(OB_FAM_GROUND, span_kernel, F, kThreads, 0, st, df, gs);
    launch(OB_FAM_GROUND, points_kernel, dim3(blocks_for(max_slots, kThreads), F), kThreads, 0, st, df, gs, pts, nflag,
           k1, u1, P, F);
    stg.check(cudaGetLastError());
    // (frame, value) order: stable sort by value, then by group (z groups 0..F-1, footprint groups F..2F-1)
    cub_run(stg, sort_pairs(k1, k2, u1, u2, static_cast<int64_t>(P2), 0, 64, st));
    cub_run(stg, sort_pairs(u2, u1, k2, k3, static_cast<int64_t>(P2), 0, bits_for(2ull * F), st));
    if (cudaError_t e = stg.error()) return fail_cuda(e, "ground points");
    launch(OB_FAM_GROUND, header_kernel, (F + 63) / 64, 64, 0, st, df, gs, static_cast<const unsigned long long*>(k3),
           P, F, grid_size);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "ground header");

    // the one host wait: the grid shapes
    std::vector<GState> hs(F);
    e = cudaMemcpyAsync(hs.data(), gs, F * sizeof(GState), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "ground grid shapes");
    unsigned long long C = 0, max_cells = 0;
    for (unsigned k = 0; k < F; ++k) {
        const ob_ground_item& it = items[slot_of[k]];
        const unsigned long long cells =
            hs[k].n_points ? static_cast<unsigned long long>(hs[k].rows) * static_cast<unsigned long long>(hs[k].cols)
                           : 0ull;
        const bool grids = it.valid || it.obstacle || it.floor_z || it.height || it.roughness;
        if (grids && cells > it.grid_capacity) return fail(OB_INVALID_ARGUMENT, "output capacity too small");
        frames[k].cell_off = C;
        C += cells;
        max_cells = std::max(max_cells, cells);
    }
    if (C >= 0x7fffffffull) return fail(OB_INVALID_ARGUMENT, "ground grid too large");
    e = cudaMemcpyAsync(df, frames.data(), F * sizeof(GFrame), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return fail_cuda(e, "ground grid offsets");
    const uint32_t nC = static_cast<uint32_t>(C);

    // grids: the model, a second (Jacobi) copy of valid / height / roughness, and the pass scratch
    Grid g{}, g2{};
    g.valid = stg.scratch<uint8_t>(C + 1);
    g.obstacle = stg.scratch<uint8_t>(C + 1);
    g.floor_z = stg.scratch<double>(C + 1);
    g.height = stg.scratch<double>(C + 1);
    g.rough = stg.scratch<double>(C + 1);
    g2.valid = stg.scratch<uint8_t>(C + 1);
    g2.height = stg.scratch<double>(C + 1);
    g2.rough = stg.scratch<double>(C + 1);
    g2.obstacle = g.obstacle;
    g2.floor_z = g.floor_z;
    auto* cbeg = stg.scratch<uint32_t>(C + 1);
    auto* cend = stg.scratch<uint32_t>(C + 1);
    auto* zs = stg.scratch<double>(P);
    auto* fz = stg.scratch<double>(P);
    auto* flags = stg.scratch<uint32_t>(P + 1);
    auto* scan = stg.scratch<uint32_t>(P + 1);
    auto* ck = stg.scratch<uint32_t>(P);
    e = stg.error();
    if (e == cudaSuccess) e = cudaMemsetAsync(cbeg, 0, (C + 1) * 4, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(cend, 0, (C + 1) * 4, st);
    if (e != cudaSuccess) return fail_cuda(e, "ground grids");
    const dim3 cgrid(blocks_for(max_cells, kThreads), F), pgrid(blocks_for(max_slots, kThreads), F);
    const unsigned flat = blocks_for(P, kThreads);

    // pass 3: cells.  Sort the slots by (cell, z): by z (the zkeys still lie in k1[0, P)), then stably by cell
    uint32_t* slots = u1;        // iota
    uint32_t* zslots = u2;       // slots by z
    uint32_t* ck_z = u1 + P;     // cell key of each z-sorted slot
    uint32_t* ck_sorted = u2 + P;
    uint32_t* cslots = u1;       // slots by (cell, z)
    launch(OB_FAM_GROUND, cell_keys_kernel, pgrid, kThreads, 0, st, df, gs, pts, k1, ck, slots, nC);
    stg.check(cudaGetLastError());
    if (cub_run(stg, sort_pairs(k1, k2, slots, zslots, static_cast<int64_t>(P), 0, 64, st)) == cudaSuccess) {
        launch(OB_FAM_GROUND, gather_kernel, flat, kThreads, 0, st, ck, zslots, ck_z, P);
        stg.check(cudaGetLastError());
    }
    cub_run(stg, sort_pairs(ck_z, ck_sorted, zslots, cslots, static_cast<int64_t>(P), 0, bits_for(C), st));
    e = stg.error();
    if (e == cudaSuccess) e = cudaMemsetAsync(flags + P, 0, 4, st);
    if (e != cudaSuccess) return fail_cuda(e, "ground cells");
    launch(OB_FAM_GROUND, cell_segments_kernel, flat, kThreads, 0, st, ck_sorted, cslots, k1, nflag, cbeg, cend, zs,
           flags, P, nC);
    stg.check(cudaGetLastError());
    // the normals-filtered lists: a flagged subsequence of each cell's sorted segment
    cub_run(stg, exclusive_sum(flags, scan, static_cast<int64_t>(P + 1), st));
    if (cudaError_t e = stg.error()) return fail_cuda(e, "ground cells");
    launch(OB_FAM_GROUND, compact_kernel, flat, kThreads, 0, st, flags, scan, zs, fz, P);
    launch(OB_FAM_GROUND, cells_kernel, cgrid, kThreads, 0, st, df, gs, cbeg, cend, zs, scan, fz, g);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "ground cells");

    // passes 4-6: every launch runs for every stop it is part of; the Jacobi passes swap g and g2
    const dim3 fgrid(blocks_for(max_cells, kFillWarps), F);
    auto fill = [&](int radius) {
        if (radius == 6) launch(OB_FAM_GROUND, fill_kernel<6>, fgrid, kFillWarps * 32, 0, st, df,
                                static_cast<const GState*>(gs), g, g2);
        else launch(OB_FAM_GROUND, fill_kernel<3>, fgrid, kFillWarps * 32, 0, st, df, static_cast<const GState*>(gs),
                    g, g2);
        std::swap(g, g2);
    };
    auto smooth = [&]() {
        launch(OB_FAM_GROUND, smooth_kernel, cgrid, kThreads, 0, st, df, static_cast<const GState*>(gs), g, g2);
        std::swap(g, g2);
    };
    uint32_t* reach = cbeg;  // cell segments are no longer needed
    uint32_t* queue = cend;
    if (stop >= OB_GROUND_FILL1) fill(6);
    if (stop >= OB_GROUND_SMOOTH1) smooth();
    if (stop >= OB_GROUND_PRUNE) launch(OB_FAM_GROUND, prune_kernel, F, 1024, 0, st, df, gs, g, reach, queue);
    if (stop >= OB_GROUND_FILL2) fill(6);
    if (stop >= OB_GROUND_SMOOTH2) smooth();
    stg.check(cudaGetLastError());
    if (!stg.error() && stop >= OB_GROUND_COMPONENTS) {
        uint32_t* parent = cbeg;
        uint32_t* csize = cend;
        auto* hk = stg.scratch<unsigned long long>(C + 1);
        auto* hk_sorted = stg.scratch<unsigned long long>(C + 1);
        auto* cells = stg.scratch<uint32_t>(C + 1);
        auto* cells_h = stg.scratch<uint32_t>(C + 1);
        auto* cells_sorted = stg.scratch<uint32_t>(C + 1);
        auto* roots_h = stg.scratch<uint32_t>(C + 1);
        auto* roots_sorted = stg.scratch<uint32_t>(C + 1);
        auto* med = stg.scratch<double>(C + 1);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "ground components");
        launch(OB_FAM_GROUND, comp_init_kernel, cgrid, kThreads, 0, st, df, static_cast<const GState*>(gs), parent,
               csize);
        launch(OB_FAM_GROUND, comp_hook_kernel, cgrid, kThreads, 0, st, df, static_cast<const GState*>(gs), g, parent);
        launch(OB_FAM_GROUND, comp_roots_kernel, cgrid, kThreads, 0, st, df, static_cast<const GState*>(gs), g, parent,
               csize, hk, cells, nC);
        stg.check(cudaGetLastError());
        // (root, height) order: by height, then stably by root (C == 0: nothing to sort)
        if (C) cub_run(stg, sort_pairs(hk, hk_sorted, cells, cells_h, static_cast<int64_t>(C), 0, 64, st));
        if (!stg.error()) {
            launch(OB_FAM_GROUND, root_keys_kernel, blocks_for(C, kThreads), kThreads, 0, st, hk_sorted, cells_h,
                   parent, roots_h, static_cast<unsigned long long>(C), nC);
            stg.check(cudaGetLastError());
        }
        if (C)
            cub_run(stg, sort_pairs(roots_h, roots_sorted, cells_h, cells_sorted, static_cast<int64_t>(C), 0,
                                    bits_for(C), st));
        if (!stg.error()) {
            launch(OB_FAM_GROUND, comp_median_kernel, blocks_for(C, kThreads), kThreads, 0, st, df, gs, roots_sorted,
                   cells_sorted, csize, g, med, F, nC);
            launch(OB_FAM_GROUND, comp_reject_kernel, cgrid, kThreads, 0, st, df, static_cast<const GState*>(gs), g,
                   parent, csize, med);
            stg.check(cudaGetLastError());
        }
    }
    if (!stg.error() && stop >= OB_GROUND_FILL3) fill(3);
    if (!stg.error()) stg.check(cudaGetLastError());
    if (cudaError_t e = stg.error()) return fail_cuda(e, "ground passes");

    // outputs: masks (classified at the last pass, else zeroed), model headers, grids
    launch(OB_FAM_GROUND, classify_kernel, dim3(blocks_for(max_px, kThreads), F), kThreads, 0, st, df,
           static_cast<const GState*>(gs), g, stop >= OB_GROUND_FINAL ? 1 : 0);
    stg.check(cudaGetLastError());
    auto* dmodel = stg.scratch<ob_ground_model>(F);
    if (!stg.error()) {
        launch(OB_FAM_GROUND, model_kernel, (F + 63) / 64, 64, 0, st, static_cast<const GState*>(gs), dmodel, F);
        stg.check(cudaGetLastError());
    }
    // n elements of device memory src into the caller's dst, host or device
    auto copy_out = [&](auto* dst, const auto* src, size_t n) {
        if (!dst || n == 0) return;
        auto* d = stg.out(dst, n);
        if (!stg.error()) stg.check(cudaMemcpyAsync(d, src, n * sizeof(*src), cudaMemcpyDeviceToDevice, st));
    };
    for (unsigned k = 0; k < F && !stg.error(); ++k) {
        const ob_ground_item& it = items[slot_of[k]];
        const size_t cells = hs[k].n_points ? static_cast<size_t>(hs[k].rows) * hs[k].cols : 0;
        const size_t off = frames[k].cell_off;
        copy_out(it.model, dmodel + k, 1);
        if (batch_of[k] >= 0) copy_out(it.vertical_subtent_out, batches[batch_of[k]].subtent + index_in_batch[k], 1);
        copy_out(it.valid, g.valid + off, cells);
        copy_out(it.obstacle, g.obstacle + off, cells);
        copy_out(it.floor_z, g.floor_z + off, cells);
        copy_out(it.height, g.height + off, cells);
        copy_out(it.roughness, g.rough + off, cells);
        copy_out(it.prune_levels, &gs[k].prune_levels, 1);
    }
    if (cudaError_t e = stg.finish()) return fail_cuda(e, "ground outputs");
    return OB_OK;
}
