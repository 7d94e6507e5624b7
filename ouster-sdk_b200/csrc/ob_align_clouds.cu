// ob_align_clouds.cu -- global cloud alignment (DESIGN f-14): the point-cloud overloads of algorithm::align_clouds,
// a yaw search by BEV cross-correlation followed by three ICP passes and an overlap confidence.
//
// What it replaces (reference paths relative to the reference tree, ouster-sdk 1.0.1):
//   features of a point cloud                    ouster_algorithm/src/align_clouds.cpp:396-454, 805-882
//   choose_xy_matcher_params, make_xy_grid_spec  :456-508, 892-904
//   build_xy_bev_grid, normalize_zero_mean_unit_norm, fft2d_inplace, align_xy_2d_fft   :906-1181
//   compute_translation_histogram, best_translation_shift, align_translation_1d       :1203-1298
//   make_confidence_sample_mask, SpatialHashGridXY, xy_matching_confidence            :237-291, 1304-1477
//   initial_pairwise_alignment, align_clouds_from_features_impl                       :1496-1581, 1893-1950
// The CPU oracle (oracle/orc_align_clouds.c) states the same operations in the same order.
//
// One call, all on the stream:
//   features     per cloud: order-preserving compaction of the valid rows (normals normalised; ob_lookback.cuh),
//                then ob_voxel_downsample at 0.4 m (AVERAGE_POINT, or POINT_NORMAL) with device counts; point
//                distances, and sorted order-preserving uint64 keys of max(|x|, |y|) and of z (the 95th-percentile
//                footprint and the floor band are order statistics, so they are exact).
//   the wait     the feature counts, footprints and guess come to the host: they size the grids and launches.
//   binsum       every BEV grid and Z histogram is a sum per cell of per-point weights: the (cell, row) items are
//                radix-sorted (stable, so a cell's rows stay in row order) and one thread sums each cell's run from
//                zero in that order, as the reference's loop does.  No floating-point atomics, so grids are
//                bit-exact and replays bit-identical.
//   Z shift      the yaw search rotates about z only, so every candidate sees the same z = z + t_z: the moving Z
//                histogram, its shift and the BEV floor / ceiling band are the same for all 187 candidates and are
//                computed once (the oracle computes them per candidate and gets the same bits).
//   pass 1       180 yaws in groups of kGroup: poses, BEV items, binsum, zero-mean / unit-norm statistics, then the
//                correlation by hand-written radix-2 FFTs in shared memory: forward rows (normalisation fused into the
//                load, rows past base_n are zero and skipped), per column forward, conj(M) T product, inverse; the
//                inverse rows only for the rows of the shift window; the window's arg-max in dy-then-dx order with
//                the first maximum kept.  Twiddles come from one host-computed table (the oracle's formula), and
//                butterflies use __d*_rn, so a transform gives the oracle's bits for the oracle's input.
//   pass 2       7 yaws on the fine grid, the same steps; the best candidate's pose with its shifts.
//   ICP          three ob_cloud_align calls (2.0, 0.6, 0.25 m) with device guess and pose.
//   confidence   the XY neighbour search is ob_cloud_nearest on z-flattened rows: with every z = 0 its 27-cell
//                search visits exactly the 9 XY cells in dx-then-dy order and its squared distance is the XY one;
//                clouds over 16 000 features are sampled by ob_voxel_downsample (SHUFFLE_FIRST); counts are integers.
//
// Scratch is taken once and reused by every group and both passes, so it does not grow with the yaw count.  Worst case
// (60 m bound: fine 481 / 1024, coarse 241 / 512), besides O(points) buffers: the two target spectra (16.8 + 4.2 MB)
// and one group's grids, spectra and windows, max(kGroup = 30 coarse yaws x 4.9 MB, 7 fine yaws x 19.5 MB) = 146 MB;
// the BEV items of a group take 24 bytes x 30 x the source feature count, plus the radix sort's temporary storage.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cuda/std/utility>

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <memory>

#include "ob_api_common.h"
#include "ob_cub.cuh"
#include "ob_lookback.cuh"
#include "ob_rows.cuh"
#include "ob_se3.cuh"

namespace ob {
namespace {

constexpr int kCoarseYaws = OB_ALIGN_COARSE_YAWS;
constexpr int kFineYaws = OB_ALIGN_FINE_YAWS;
constexpr int kYaws = kCoarseYaws + kFineYaws;
constexpr int kZBins = OB_ALIGN_Z_BINS;
constexpr int kZFft = 2048;       // next_power_of_two(2 * 1024 - 1)
constexpr int kZMaxShift = 20;    // llround(4.0 / 0.2)
constexpr int kTwN = 2048;        // the twiddle table's transform size; smaller sizes take every (2048 / n)-th entry
constexpr int kGroup = 30;        // pass-1 yaws per group
constexpr unsigned kThreads = 256;
constexpr double kPi = 3.14159265358979323846;
constexpr double kNormalEps = 1e-12;
constexpr double kVoxel = 0.4;
constexpr double kPitch = 0.2;
constexpr double kCoarsePixel = 0.5;
constexpr size_t kMinPoints = 20;
constexpr unsigned kConfSamples = 16000;

// ---- device state of one call ----
struct Filter {  // build_xy_bev_grid's floor / ceiling band
    int on;
    double floor_cut, ceil_cut;
};
struct Probe {  // what the one wait reads
    unsigned long long nf[2];  // feature counts: source, target
    double foot[2];            // 95th-percentile footprints
    double guess[16];          // initial_guess (identity for none)
};
struct State {
    Probe probe;
    double zstat[2][3];   // zmin, zmax, 4th-percentile z of the source and target features
    Filter filt_t, filt_s;
    int zbins;            // the Z shift in bins
    int coarse_index, fine_index, pad;
    double dz;            // clipped Z shift (m)
    double scores[kYaws];
    int dx[kYaws], dy[kYaws];
    double cand[kYaws][16];  // candidate poses (before the XY shift)
    double initial_pose[16];
    double icp[3][16];
    unsigned long long counts[2][4];  // [initial, refined][source total, source matched, target total, matched]
    double conf[2];
    int target_valid[2];  // fine, coarse: the target grid is not empty
};

__device__ Filter filter_of(const double* zs, double c) {
    // order statistics of z + c are those of z, plus c (x -> x + c is monotone in floating point)
    const double lo = add(zs[0], c), hi = add(zs[1], c), range = sub(hi, lo);
    Filter f;
    f.on = isfinite(range) && range > 1.0;
    f.floor_cut = add(f.on ? add(zs[2], c) : lo, 0.2);
    f.ceil_cut = sub(hi, 0.1);
    return f;
}

// ---- features ----
// valid rows (finite point; with normals a finite normal of norm > 1e-12, normalised) in row order
template <typename T>
__global__ void __launch_bounds__(kThreads) ac_valid_kernel(Rows r, const void* nrm, unsigned* ticket, Lookback lb,
                                                            double* op, double* on, unsigned long long* count) {
    using BS = cub::BlockScan<unsigned, kThreads>;
    __shared__ typename BS::TempStorage tmp;
    __shared__ unsigned s_bid;
    __shared__ unsigned long long s_excl;
    if (threadIdx.x == 0) s_bid = atomicAdd(ticket, 1u);
    __syncthreads();
    const unsigned bid = s_bid;
    const unsigned i = bid * kThreads + threadIdx.x;
    double p[3], q[3];
    bool ok = false;
    if (i < rows_n(r)) {
        load3<T>(r.p, i, p);
        ok = finite3(p);
        if (ok && nrm) {
            load3<T>(nrm, i, q);
            const double len = norm3(q);
            ok = finite3(q) && len > kNormalEps;
            for (int d = 0; d < 3; ++d) q[d] = q[d] / len;
        }
    }
    unsigned rank, total;
    BS(tmp).ExclusiveSum(ok ? 1u : 0u, rank, total);
    if (threadIdx.x < 32) {
        const unsigned long long excl = lookback_exclusive(lb, bid, total, threadIdx.x);
        if (threadIdx.x == 0) {
            s_excl = excl;
            if (bid + 1 == gridDim.x) *count = excl + total;
        }
    }
    __syncthreads();
    if (!ok) return;
    const size_t o = s_excl + rank;
    for (int d = 0; d < 3; ++d) {
        op[3 * o + d] = p[d];
        if (nrm) on[3 * o + d] = q[d];
    }
}

// point_dist and the sort keys of the footprint and z percentiles; rows past the count get keys that sort last
__global__ void ac_keys_kernel(const double* fp, const unsigned long long* nf, unsigned cap, double* dist,
                               unsigned long long* ekey, unsigned long long* zkey) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    if (i >= *nf) {
        ekey[i] = zkey[i] = ~0ull;
        return;
    }
    const double* p = fp + 3 * static_cast<size_t>(i);
    dist[i] = norm3(p);
    ekey[i] = okey(smax(fabs(p[0]), fabs(p[1])));
    zkey[i] = okey(p[2]);
}

// footprints (estimate_xy_footprint_bound), z statistics, the target's band, the guess
__global__ void ac_stats_kernel(const unsigned long long* nf_s, const unsigned long long* nf_t,
                                const unsigned long long* eks, const unsigned long long* ekt,
                                const unsigned long long* zks, const unsigned long long* zkt, const double* guess,
                                State* st) {
    const unsigned long long n[2] = {*nf_s, *nf_t};
    const unsigned long long* ek[2] = {eks, ekt};
    const unsigned long long* zk[2] = {zks, zkt};
    for (int c = 0; c < 2; ++c) {
        st->probe.nf[c] = n[c];
        st->probe.foot[c] = 10.0;
        if (n[c] == 0) continue;
        st->probe.foot[c] = okey_value(ek[c][static_cast<size_t>(floor(mul(0.95, static_cast<double>(n[c] - 1))))]);
        size_t p = static_cast<size_t>(mul(0.04, static_cast<double>(n[c])));
        if (p > n[c] - 1) p = n[c] - 1;
        st->zstat[c][0] = okey_value(zk[c][0]);
        st->zstat[c][1] = okey_value(zk[c][n[c] - 1]);
        st->zstat[c][2] = okey_value(zk[c][p]);
    }
    for (int j = 0; j < 16; ++j) st->probe.guess[j] = guess ? guess[j] : (j % 5 == 0 ? 1.0 : 0.0);
    st->filt_t = filter_of(st->zstat[1], 0.0);
}

// ---- binsum: per-cell sums in row order ----
struct BevSpec {
    double half, inv;  // bound, 1 / pixel
    int base_n;
};

// one item per (candidate, feature row): its cell (or `total` when dropped) and weight.  kZ: the Z histogram
// (compute_translation_histogram along UnitZ); else the BEV grid (build_xy_bev_grid).  poses null: the features as
// they are (the target); else candidate g's pose poses[16 g] (the source).
template <bool kZ>
__global__ void ac_items_kernel(const double* fp, const double* fn, const double* dist, unsigned n,
                                const double* poses, BevSpec bs, const Filter* filt, uint32_t total, uint32_t* keys,
                                uint32_t* vals, double* w) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned g = blockIdx.y;
    const size_t item = static_cast<size_t>(g) * n + i;
    keys[item] = total;
    vals[item] = static_cast<uint32_t>(item);
    w[item] = 0.0;
    const double di = dist[i];
    if (di <= 0.0) return;
    double x[3], m[3];
    const double* p = fp + 3 * static_cast<size_t>(i);
    const double* q = fn ? fn + 3 * static_cast<size_t>(i) : nullptr;
    if (poses) {
        mat4_transform(poses + 16 * g, p, x);
        if (q) mat4_rotate(poses + 16 * g, q, m);
    } else {
        for (int d = 0; d < 3; ++d) {
            x[d] = p[d];
            if (q) m[d] = q[d];
        }
    }
    double wt = 1.0;
    if (kZ) {
        if (q) {
            wt = fabs(add(add(mul(m[0], 0.0), mul(m[1], 0.0)), mul(m[2], 1.0)));
            if (wt <= 0.5) return;
        }
        const double z = add(add(mul(x[0], 0.0), mul(x[1], 0.0)), mul(x[2], 1.0));
        const long long pos = llround(z / kPitch) + kZBins / 2;
        if (pos < 0 || pos >= kZBins) return;
        keys[item] = static_cast<uint32_t>(pos);
        w[item] = mul(wt, di);
        return;
    }
    if (!finite3(x)) return;
    if (filt->on && (x[2] <= filt->floor_cut || x[2] >= filt->ceil_cut)) return;
    if (fabs(x[0]) > bs.half || fabs(x[1]) > bs.half) return;
    wt = di;
    if (q) {
        if (!finite3(m)) return;
        const double strength = add(mul(m[0], m[0]), mul(m[1], m[1]));
        if (strength < 0.5) return;
        wt = mul(wt, strength);
    }
    const double fx = floor(mul(add(x[0], bs.half), bs.inv)), fy = floor(mul(add(x[1], bs.half), bs.inv));
    if (fx < 0.0 || fy < 0.0 || fx >= bs.base_n || fy >= bs.base_n) return;
    const unsigned cells = static_cast<unsigned>(bs.base_n) * bs.base_n;
    keys[item] = g * cells + static_cast<unsigned>(fy) * bs.base_n + static_cast<unsigned>(fx);
    w[item] = wt;
}

// one thread per run of equal keys: its weights summed from zero in row order
__global__ void ac_segsum_kernel(const uint32_t* sk, const uint32_t* sv, const double* w, size_t items,
                                 uint32_t total, double* out) {
    const size_t q = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (q >= items) return;
    const uint32_t k = sk[q];
    if (k >= total || (q > 0 && sk[q - 1] == k)) return;
    double acc = 0.0;
    for (size_t p = q; p < items && sk[p] == k; ++p) acc = add(acc, w[sv[p]]);
    out[k] = acc;
}

// ---- normalisation statistics: mean and norm after the mean, one block per grid ----
__global__ void __launch_bounds__(kThreads) ac_norm_kernel(const double* grids, unsigned cells, double* mean,
                                                           double* rn, int* valid) {
    using BR = cub::BlockReduce<double, kThreads>;
    __shared__ typename BR::TempStorage tmp;
    __shared__ double s_mean;
    const double* g = grids + static_cast<size_t>(blockIdx.x) * cells;
    double s = 0.0;
    for (unsigned i = threadIdx.x; i < cells; i += kThreads) s = add(s, g[i]);
    s = BR(tmp).Sum(s);
    if (threadIdx.x == 0) s_mean = s / static_cast<double>(cells);
    __syncthreads();
    const double mu = s_mean;
    double v = 0.0;
    for (unsigned i = threadIdx.x; i < cells; i += kThreads) {
        const double d = sub(g[i], mu);
        v = add(v, mul(d, d));
    }
    __syncthreads();
    v = BR(tmp).Sum(v);
    if (threadIdx.x == 0) {
        mean[blockIdx.x] = mu;
        const bool ok = isfinite(v) && v > 1e-30;  // normalize_zero_mean_unit_norm; else the grid counts as empty
        rn[blockIdx.x] = ok ? sqrt(v) : 1.0;
        valid[blockIdx.x] = ok;
    }
}

// ---- radix-2 FFT in shared memory ----
__device__ __forceinline__ unsigned bitrev(unsigned i, unsigned logn) { return __brev(i) >> (32 - logn); }

// in place on bit-reversed data; tw[k] = exp(-2 pi i k / kTwN); the inverse conjugates and scales by 1 / n
template <bool kInv>
__device__ void fft_smem(double* re, double* im, unsigned n, const double2* __restrict__ tw) {
    for (unsigned len = 2; len <= n; len <<= 1) {
        const unsigned half = len >> 1, step = kTwN / len;
        for (unsigned b = threadIdx.x; b < n / 2; b += blockDim.x) {
            const unsigned j = b & (half - 1), i = (b / half) * len + j;
            const double2 t = tw[j * step];
            const double wr = t.x, wi = kInv ? -t.y : t.y;
            const double br = re[i + half], bi = im[i + half];
            const double vr = sub(mul(br, wr), mul(bi, wi)), vi = add(mul(br, wi), mul(bi, wr));
            const double ur = re[i], ui = im[i];
            re[i] = add(ur, vr);
            im[i] = add(ui, vi);
            re[i + half] = sub(ur, vr);
            im[i + half] = sub(ui, vi);
        }
        __syncthreads();
    }
    if (kInv) {
        const double s = 1.0 / static_cast<double>(n);
        for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
            re[i] = mul(re[i], s);
            im[i] = mul(im[i], s);
        }
        __syncthreads();
    }
}

struct FftShape {
    unsigned bn, n, logn, ms;  // base_n, fft_n, log2(fft_n), window half-width
};

// forward transform of rows y < base_n of grid blockIdx.y, normalised on load: spec[grid][y][n]
__global__ void __launch_bounds__(kThreads) ac_fft_rows_kernel(const double* grids, FftShape f, const double* mean,
                                                               const double* rn, const double2* tw, double2* spec) {
    extern __shared__ double sm[];
    double *re = sm, *im = sm + f.n;
    const unsigned c = blockIdx.y, y = blockIdx.x;
    const double* g = grids + (static_cast<size_t>(c) * f.bn + y) * f.bn;
    const double mu = mean[c], r = rn[c];
    for (unsigned i = threadIdx.x; i < f.n; i += blockDim.x) {
        const unsigned j = bitrev(i, f.logn);
        re[j] = i < f.bn ? sub(g[i], mu) / r : 0.0;
        im[j] = 0.0;
    }
    __syncthreads();
    fft_smem<false>(re, im, f.n, tw);
    double2* o = spec + (static_cast<size_t>(c) * f.bn + y) * f.n;
    for (unsigned i = threadIdx.x; i < f.n; i += blockDim.x) o[i] = make_double2(re[i], im[i]);
}

// column blockIdx.x of grid blockIdx.y: forward transform (rows >= base_n are zero).  kTarget: store the column
// (out[col][row]).  Else: times conj(M) T, inverse transform, and the window rows out[grid][dy + ms][col].
template <bool kTarget>
__global__ void __launch_bounds__(kThreads) ac_fft_cols_kernel(const double2* spec, FftShape f, const double2* tw,
                                                               const double2* tspec, double2* out) {
    extern __shared__ double sm[];
    double *re = sm, *im = sm + f.n;
    const unsigned c = blockIdx.y, col = blockIdx.x;
    const double2* s = spec + static_cast<size_t>(c) * f.bn * f.n + col;
    for (unsigned y = threadIdx.x; y < f.n; y += blockDim.x) {
        const unsigned j = bitrev(y, f.logn);
        const double2 v = y < f.bn ? s[static_cast<size_t>(y) * f.n] : make_double2(0.0, 0.0);
        re[j] = v.x;
        im[j] = v.y;
    }
    __syncthreads();
    fft_smem<false>(re, im, f.n, tw);
    if constexpr (kTarget) {
        double2* o = out + static_cast<size_t>(col) * f.n;
        for (unsigned y = threadIdx.x; y < f.n; y += blockDim.x) o[y] = make_double2(re[y], im[y]);
        return;
    }
    const double2* t = tspec + static_cast<size_t>(col) * f.n;
    // product, written back in bit-reversed order for the inverse
    double pr[8], pi[8];  // n <= 1024 = 4 x 256 threads
    unsigned k = 0;
    for (unsigned y = threadIdx.x; y < f.n; y += blockDim.x, ++k) {
        const double mr = re[y], mi = im[y];
        const double2 tv = t[y];
        pr[k] = add(mul(mr, tv.x), mul(mi, tv.y));
        pi[k] = sub(mul(mr, tv.y), mul(mi, tv.x));
    }
    __syncthreads();
    k = 0;
    for (unsigned y = threadIdx.x; y < f.n; y += blockDim.x, ++k) {
        const unsigned j = bitrev(y, f.logn);
        re[j] = pr[k];
        im[j] = pi[k];
    }
    __syncthreads();
    fft_smem<true>(re, im, f.n, tw);
    const unsigned W = 2 * f.ms + 1;
    double2* o = out + static_cast<size_t>(c) * W * f.n + col;
    for (unsigned w = threadIdx.x; w < W; w += blockDim.x) {
        const int dy = static_cast<int>(w) - static_cast<int>(f.ms);
        const unsigned y = dy >= 0 ? static_cast<unsigned>(dy) : f.n - static_cast<unsigned>(-dy);
        o[static_cast<size_t>(w) * f.n] = make_double2(re[y], im[y]);
    }
}

// inverse transform of window row blockIdx.x of grid blockIdx.y; the real parts of the window's columns
__global__ void __launch_bounds__(kThreads) ac_fft_window_kernel(const double2* rows, FftShape f, const double2* tw,
                                                                 double* win) {
    extern __shared__ double sm[];
    double *re = sm, *im = sm + f.n;
    const unsigned W = 2 * f.ms + 1;
    const unsigned c = blockIdx.y, w = blockIdx.x;
    const double2* r = rows + (static_cast<size_t>(c) * W + w) * f.n;
    for (unsigned i = threadIdx.x; i < f.n; i += blockDim.x) {
        const unsigned j = bitrev(i, f.logn);
        const double2 v = r[i];
        re[j] = v.x;
        im[j] = v.y;
    }
    __syncthreads();
    fft_smem<true>(re, im, f.n, tw);
    double* o = win + (static_cast<size_t>(c) * W + w) * W;
    for (unsigned k = threadIdx.x; k < W; k += blockDim.x) {
        const int dx = static_cast<int>(k) - static_cast<int>(f.ms);
        o[k] = re[dx >= 0 ? static_cast<unsigned>(dx) : f.n - static_cast<unsigned>(-dx)];
    }
}

using Peak = cuda::std::pair<double, int>;  // value, window index (dy-major)
struct FirstMax {
    __device__ Peak operator()(const Peak& a, const Peak& b) const {
        return (b.first > a.first || (b.first == a.first && b.second < a.second)) ? b : a;
    }
};

// the window's best score, scanning dy then dx and keeping the first strictly greater value (align_xy_2d_fft);
// 0 at (0, 0) for an empty moving or target grid.  Results at candidate first + blockIdx.x.
__global__ void __launch_bounds__(kThreads) ac_argmax_kernel(const double* win, unsigned ms, const int* valid,
                                                             const int* target_valid, int first, State* st) {
    using BR = cub::BlockReduce<Peak, kThreads>;
    __shared__ typename BR::TempStorage tmp;
    const unsigned W = 2 * ms + 1, c = blockIdx.x;
    const double* v = win + static_cast<size_t>(c) * W * W;
    Peak best{-DBL_MAX, INT_MAX};
    for (unsigned i = threadIdx.x; i < W * W; i += blockDim.x)
        if (v[i] > best.first) best = Peak(v[i], static_cast<int>(i));
    best = BR(tmp).Reduce(best, FirstMax());
    if (threadIdx.x != 0) return;
    const int k = first + static_cast<int>(c);
    if (!valid[c] || !*target_valid) {
        st->scores[k] = 0.0;
        st->dx[k] = st->dy[k] = 0;
        return;
    }
    st->scores[k] = best.first;
    st->dx[k] = best.second == INT_MAX ? 0 : best.second % static_cast<int>(W) - static_cast<int>(ms);
    st->dy[k] = best.second == INT_MAX ? 0 : best.second / static_cast<int>(W) - static_cast<int>(ms);
}

// ---- Z shift (best_translation_shift over 2048-point transforms), once for every candidate ----
__global__ void __launch_bounds__(kThreads) ac_zshift_kernel(const double* hm, const double* ht, const double2* tw,
                                                             double g23, State* st) {
    __shared__ double ar[kZFft], ai[kZFft];
    constexpr unsigned logn = 11, kPer = kZFft / kThreads;
    double tr[kPer], ti[kPer], pr[kPer], pi[kPer];
    // the target's transform first, kept in registers
    for (unsigned i = threadIdx.x; i < kZFft; i += blockDim.x) {
        const unsigned j = bitrev(i, logn);
        ar[j] = i < kZBins ? ht[i] : 0.0;
        ai[j] = 0.0;
    }
    __syncthreads();
    fft_smem<false>(ar, ai, kZFft, tw);
    unsigned k = 0;
    for (unsigned i = threadIdx.x; i < kZFft; i += blockDim.x, ++k) {
        tr[k] = ar[i];
        ti[k] = ai[i];
    }
    __syncthreads();
    for (unsigned i = threadIdx.x; i < kZFft; i += blockDim.x) {
        const unsigned j = bitrev(i, logn);
        ar[j] = i < kZBins ? hm[i] : 0.0;
        ai[j] = 0.0;
    }
    __syncthreads();
    fft_smem<false>(ar, ai, kZFft, tw);
    k = 0;
    for (unsigned i = threadIdx.x; i < kZFft; i += blockDim.x, ++k) {
        pr[k] = add(mul(ar[i], tr[k]), mul(ai[i], ti[k]));
        pi[k] = sub(mul(ar[i], ti[k]), mul(ai[i], tr[k]));
    }
    __syncthreads();
    k = 0;
    for (unsigned i = threadIdx.x; i < kZFft; i += blockDim.x, ++k) {
        const unsigned j = bitrev(i, logn);
        ar[j] = pr[k];
        ai[j] = pi[k];
    }
    __syncthreads();
    fft_smem<true>(ar, ai, kZFft, tw);
    if (threadIdx.x != 0) return;
    int best_shift = 0;
    double best = -DBL_MAX;
    for (int s = -kZMaxShift; s <= kZMaxShift; ++s) {
        const double v = ar[s >= 0 ? s : kZFft + s];
        if (v > best) {
            best = v;
            best_shift = s;
        }
    }
    st->zbins = best_shift;
    st->dz = smax(-4.0, smin(mul(kPitch, static_cast<double>(best_shift)), 4.0));
    st->filt_s = filter_of(st->zstat[0], add(g23, st->dz));
}

// ---- candidate poses: PoseH(RotV(0, 0, yaw).exp()) * G, then the Z shift ----
// pass 1: yaws first .. first + count - 1; pass 2 (first < 0): the 7 fine yaws around the coarse pick.  The yaw
// rotations come from a host table (yaw_table), so they carry host libm's sin / cos bits, as the oracle's do.
__global__ void ac_pose_kernel(int first, int count, const double* yaw_table, const double* G, State* st) {
    const int k = static_cast<int>(threadIdx.x);
    if (k >= count) return;
    const int slot = first >= 0 ? first + k : kCoarseYaws + k;
    const int row = first >= 0 ? first + k : kCoarseYaws + st->coarse_index * kFineYaws + k;
    mat4_mul(yaw_table + 16 * row, G, st->cand[slot]);
    st->cand[slot][11] = add(st->cand[slot][11], st->dz);
}

// the best coarse yaw (first strictly greater score)
__global__ void ac_coarse_pick_kernel(State* st) {
    int best = -1;
    double s = -DBL_MAX;
    for (int i = 0; i < kCoarseYaws; ++i)
        if (st->scores[i] > s) {
            s = st->scores[i];
            best = i;
        }
    st->coarse_index = best < 0 ? 0 : best;
}

// the best fine candidate's pose with its XY shift (G when no score beats lowest())
__global__ void ac_fine_pick_kernel(const double* G, double pixel, State* st) {
    double s = -DBL_MAX;
    st->fine_index = -1;
    for (int j = 0; j < 16; ++j) st->initial_pose[j] = G[j];
    for (int k = 0; k < kFineYaws; ++k) {
        const int c = kCoarseYaws + k;
        if (!(st->scores[c] > s)) continue;
        s = st->scores[c];
        st->fine_index = k;
        for (int j = 0; j < 16; ++j) st->initial_pose[j] = st->cand[c][j];
        st->initial_pose[3] = add(st->initial_pose[3], mul(pixel, static_cast<double>(st->dx[c])));
        st->initial_pose[7] = add(st->initial_pose[7], mul(pixel, static_cast<double>(st->dy[c])));
    }
}

// ---- confidence ----
// query rows of one direction at pose P (inverse: R^T p - R^T t), z flattened; `flat` = the rows, z flattened
__global__ void ac_query_kernel(const double* fp, const unsigned long long* nf, unsigned cap, const double* P,
                                int inverse, double* q) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap || i >= *nf) return;
    const double* p = fp + 3 * static_cast<size_t>(i);
    double x[2];
    if (P == nullptr) {
        x[0] = p[0];
        x[1] = p[1];
    } else {
        for (int d = 0; d < 2; ++d) {
            if (!inverse) {
                x[d] = add(add(add(mul(P[4 * d], p[0]), mul(P[4 * d + 1], p[1])), mul(P[4 * d + 2], p[2])), P[4 * d + 3]);
            } else {  // Ri = R^T, ti = (-Ri) t
                const double ti = add(add(mul(-P[d], P[3]), mul(-P[4 + d], P[7])), mul(-P[8 + d], P[11]));
                x[d] = add(add(add(mul(P[d], p[0]), mul(P[4 + d], p[1])), mul(P[8 + d], p[2])), ti);
            }
        }
    }
    q[3 * static_cast<size_t>(i)] = x[0];
    q[3 * static_cast<size_t>(i) + 1] = x[1];
    q[3 * static_cast<size_t>(i) + 2] = 0.0;
}

// make_confidence_sample_mask: with idx, the first 16 000 rows of the shuffled downsample (mask zeroed before);
// without, every row
__global__ void ac_mask_kernel(const uint32_t* idx, const unsigned long long* count, unsigned cap, uint8_t* mask) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    if (!idx) mask[i] = i < *count ? 1 : 0;
    else if (i < kConfSamples && i < *count) mask[idx[i]] = 1;
}

// count_direction: total = sampled finite query rows, matched = those with an XY neighbour (and, with normals, a
// rotated normal within 5 degrees of the neighbour's)
__global__ void __launch_bounds__(kThreads) ac_count_kernel(const double* qn, const unsigned long long* nf, unsigned cap,
                                                            const uint8_t* mask, const int32_t* nn, const double* gn,
                                                            const double* P, int inverse, double cos_gate,
                                                            unsigned long long* out) {
    using BR = cub::BlockReduce<unsigned, kThreads>;
    __shared__ typename BR::TempStorage tmp;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned t = 0, m = 0;
    if (i < cap && i < *nf && mask[i]) {
        t = 1;
        const int j = nn[i];
        if (j >= 0) {
            if (!qn) {
                m = 1;
            } else {
                double a[3], b[3], w[3];
                for (int d = 0; d < 3; ++d) {
                    a[d] = qn[3 * static_cast<size_t>(i) + d];
                    b[d] = gn[3 * static_cast<size_t>(j) + d];
                }
                const double an = norm3(a), bn = norm3(b);
                if (finite3(a) && finite3(b) && an > kNormalEps && bn > kNormalEps) {
                    for (int d = 0; d < 3; ++d) {
                        a[d] = a[d] / an;
                        b[d] = b[d] / bn;
                    }
                    for (int d = 0; d < 3; ++d)
                        w[d] = inverse ? add(add(mul(P[d], a[0]), mul(P[4 + d], a[1])), mul(P[8 + d], a[2]))
                                       : add(add(mul(P[4 * d], a[0]), mul(P[4 * d + 1], a[1])), mul(P[4 * d + 2], a[2]));
                    const double wsq = sqn3(w[0], w[1], w[2]);
                    if (wsq > 0.0) {
                        const double wn = sqrt(wsq);
                        for (int d = 0; d < 3; ++d) w[d] = w[d] / wn;
                    }
                    m = fabs(add(add(mul(w[0], b[0]), mul(w[1], b[1])), mul(w[2], b[2]))) >= cos_gate ? 1 : 0;
                }
            }
        }
    }
    const unsigned bt = BR(tmp).Sum(t);
    __syncthreads();
    const unsigned bm = BR(tmp).Sum(m);
    if (threadIdx.x == 0) {
        atomicAdd(out, static_cast<unsigned long long>(bt));
        atomicAdd(out + 1, static_cast<unsigned long long>(bm));
    }
}

__device__ double conf_of(const unsigned long long* c) {
    if (c[0] == 0 || c[2] == 0) return 0.0;
    const double v = static_cast<double>(c[1] + c[3]) / static_cast<double>(c[0] + c[2]);
    return !isfinite(v) ? 0.0 : (v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v));
}

// the guard (refined + 1e-6 < initial: the initial pose) and the outputs
__global__ void ac_finish_kernel(State* st, int compute_confidence, double* pose, double* confidence) {
    const double ci = conf_of(st->counts[0]);
    double cr = conf_of(st->counts[1]);
    st->conf[0] = ci;
    st->conf[1] = cr;
    const double* p = st->icp[2];
    if (add(cr, 1e-6) < ci) {
        p = st->initial_pose;
        cr = ci;
    }
    for (int j = 0; j < 16; ++j) pose[j] = p[j];
    if (confidence) *confidence = compute_confidence ? cr : 0.0;
}

// ---- host side ----
unsigned nblocks(size_t n) { return static_cast<unsigned>(std::max<size_t>(1, (n + kThreads - 1) / kThreads)); }

// RotV(0, 0, yaw).exp() as a 4 x 4 with zero translation (PoseV::exp, transform_vector.cpp:40-60, in the oracle's
// order of evaluation): the 180 coarse yaws, then the 7 fine yaws around each of them
void yaw_delta(double yaw, double* D) {
    const double v[3] = {0.0, 0.0, yaw};
    const double angle = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    const double sa = std::sin(angle), ca = std::cos(angle);
    double R[3][3];
    auto skew = [](const double* w, double m[3][3]) {
        m[0][0] = 0.0, m[0][1] = -w[2], m[0][2] = w[1];
        m[1][0] = w[2], m[1][1] = 0.0, m[1][2] = -w[0];
        m[2][0] = -w[1], m[2][1] = w[0], m[2][2] = 0.0;
    };
    if (angle < std::sqrt(DBL_EPSILON)) {
        double sk[3][3];
        skew(v, sk);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i][j] = (i == j ? 1.0 : 0.0) + sk[i][j];
    } else {
        const double ax[3] = {v[0] / angle, v[1] / angle, v[2] / angle};
        double a[3][3], b[3][3], bb[3][3];
        skew(ax, a);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) b[i][j] = (1.0 - ca) * a[i][j];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) bb[i][j] = (b[i][0] * a[0][j] + b[i][1] * a[1][j]) + b[i][2] * a[2][j];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i][j] = ((i == j ? 1.0 : 0.0) + sa * a[i][j]) + bb[i][j];
    }
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) D[4 * i + j] = R[i][j];
        D[4 * i + 3] = 0.0;
    }
    D[12] = D[13] = D[14] = 0.0;
    D[15] = 1.0;
}

const double* yaw_table() {
    static const std::vector<double> t = [] {
        std::vector<double> v(16 * (kCoarseYaws + kCoarseYaws * kFineYaws));
        const double coarse_step = 2.0 * kPi / static_cast<double>(kCoarseYaws);
        const double half_range = 3.0 * kPi / 180.0, step = 1.0 * kPi / 180.0;
        for (int i = 0; i < kCoarseYaws; ++i) {
            const double best_yaw = static_cast<double>(i) * coarse_step;
            yaw_delta(best_yaw, v.data() + 16 * i);
            for (int k = 0; k < kFineYaws; ++k)
                yaw_delta(best_yaw - half_range + static_cast<double>(k) * step,
                          v.data() + 16 * (kCoarseYaws + i * kFineYaws + k));
        }
        return v;
    }();
    return t.data();
}

const double2* twiddles() {  // exp(-2 pi i k / 2048), the oracle's formula
    static const std::vector<double2> t = [] {
        std::vector<double2> v(kTwN / 2);
        for (int k = 0; k < kTwN / 2; ++k) {
            const double ang = -2.0 * kPi * static_cast<double>(k) / static_cast<double>(kTwN);
            v[k] = make_double2(std::cos(ang), std::sin(ang));
        }
        return v;
    }();
    return t.data();
}

struct Spec {  // make_xy_grid_spec plus the shift window of align_xy_2d_fft
    double pixel, bound;
    int base_n, fft_n, max_shift;
};
Spec make_spec(double pixel, double bound, double max_shift_m) {
    Spec s;
    s.pixel = std::max(1e-6, pixel);
    s.bound = std::max(s.pixel, bound);
    const double span = 2.0 * s.bound;
    s.base_n = std::max(8, static_cast<int>(std::ceil(span / s.pixel)) + 1);
    int n = 1;
    while (n < 2 * s.base_n - 1) n <<= 1;
    s.fft_n = std::max(n, 8);
    const long long bins = std::max(1LL, std::llround(std::max(0.1, max_shift_m) / s.pixel));
    s.max_shift = static_cast<int>(std::min<long long>(bins, s.base_n / 2));
    return s;
}
FftShape shape_of(const Spec& s) {
    unsigned logn = 0;
    while ((1 << logn) < s.fft_n) ++logn;
    return FftShape{static_cast<unsigned>(s.base_n), static_cast<unsigned>(s.fft_n), logn,
                    static_cast<unsigned>(s.max_shift)};
}

struct Cloud {
    Rows rows;
    const void* nrm;          // staged input normals or null
    double *vp, *vn;          // valid rows
    double *fp, *fn, *dist;   // features
    unsigned long long *nv, *nf;
    unsigned cap;
    size_t n;  // the feature count, after the wait
};

class Run {
   public:
    Run(const ob_align_clouds_io* io, ob_stream* s, Staging& stg)
        : io_(io), s_(s), st_(stream_handle(s)), stg_(stg), tw_(stg.in(twiddles(), kTwN / 2)) {}

    template <typename T>
    ob_status features(Cloud& c, const char* what);
    ob_status wait_probe(Probe* p);
    // per-cell sums of `items` = groups x n items into out (groups x cells)
    template <bool kZ>
    ob_status binsum(const Cloud& c, const double* poses, unsigned groups, const BevSpec& bs, const Filter* filt,
                     uint32_t cells, double* out);
    ob_status correlate(const Cloud& src, const Spec& sp, const double2* tspec, const int* tvalid, int first,
                        unsigned count, const Filter* filt);
    ob_status target_spectrum(const Cloud& tgt, const Spec& sp, const Filter* filt, double* grid, double2* tspec,
                              int* tvalid);
    ob_status confidence(Cloud& src, Cloud& tgt, bool normals, int which, const double* P);
    // one set of binsum and correlation buffers, sized for the largest user and reused by every group and pass
    ob_status workspace(const Cloud& src, const Cloud& tgt, const Spec& fine, const Spec& coarse);

    const ob_align_clouds_io* io_;
    ob_stream* s_;
    cudaStream_t st_;
    Staging& stg_;
    const double2* tw_;
    State* state_ = nullptr;
    uint8_t* mask_[2] = {nullptr, nullptr};
    double* flat_[2] = {nullptr, nullptr};
    double* query_[2] = {nullptr, nullptr};
    int32_t* nn_[2] = {nullptr, nullptr};
    uint32_t *keys_ = nullptr, *skeys_ = nullptr, *vals_ = nullptr, *svals_ = nullptr;
    double* w_ = nullptr;
    std::unique_ptr<CubTemp> sort_tmp_;
    double *grids_ = nullptr, *mean_ = nullptr, *rn_ = nullptr, *win_ = nullptr;
    int* valid_ = nullptr;
    double2 *spec_ = nullptr, *rows_ = nullptr;
};

ob_status Run::workspace(const Cloud& src, const Cloud& tgt, const Spec& fine, const Spec& coarse) {
    const size_t items = std::max({static_cast<size_t>(kGroup) * src.n, static_cast<size_t>(kFineYaws) * src.n, tgt.n});
    keys_ = stg_.scratch<uint32_t>(items);
    skeys_ = stg_.scratch<uint32_t>(items);
    vals_ = stg_.scratch<uint32_t>(items);
    svals_ = stg_.scratch<uint32_t>(items);
    w_ = stg_.scratch<double>(items);
    // temporary storage for the largest sort: every item, every key bit
    sort_tmp_ = std::make_unique<CubTemp>(stg_, sort_pairs(keys_, skeys_, vals_, svals_, static_cast<int>(items), 0, 32, st_));
    size_t g = 0, sp = 0, rw = 0, wn = 0;
    for (const auto& [s, count] : {std::pair<const Spec&, size_t>(coarse, kGroup), {fine, kFineYaws}}) {
        const FftShape f = shape_of(s);
        const size_t W = 2 * f.ms + 1;
        g = std::max(g, count * f.bn * f.bn);
        sp = std::max(sp, count * f.bn * f.n);
        rw = std::max(rw, count * W * f.n);
        wn = std::max(wn, count * W * W);
    }
    grids_ = stg_.scratch<double>(g);
    spec_ = stg_.scratch<double2>(sp);
    rows_ = stg_.scratch<double2>(rw);
    win_ = stg_.scratch<double>(wn);
    mean_ = stg_.scratch<double>(kGroup);
    rn_ = stg_.scratch<double>(kGroup);
    valid_ = stg_.scratch<int>(kGroup);
    const Cloud* cl[2] = {&src, &tgt};
    for (int c = 0; c < 2; ++c) {
        query_[c] = stg_.scratch<double>(cl[c]->cap * 3ull);
        nn_[c] = stg_.scratch<int32_t>(cl[c]->cap);
    }
    if (cudaError_t e = stg_.error()) return fail_cuda(e, "align clouds workspace");
    return OB_OK;
}

template <typename T>
ob_status Run::features(Cloud& c, const char* what) {
    const unsigned cap = c.cap, nb = nblocks(cap);
    c.vp = stg_.scratch<double>(cap * 3ull);
    c.vn = c.nrm ? stg_.scratch<double>(cap * 3ull) : nullptr;
    c.fp = stg_.scratch<double>(cap * 3ull);
    c.fn = c.nrm ? stg_.scratch<double>(cap * 3ull) : nullptr;
    c.dist = stg_.scratch<double>(cap);
    c.nv = stg_.scratch<unsigned long long>(1);
    c.nf = stg_.scratch<unsigned long long>(1);
    auto* b = stg_.scratch<uint8_t>(16 + nb * 4ull + 8 + nb * 16ull);
    if (cudaError_t e = stg_.error()) return fail_cuda(e, what);
    const size_t sb = 16 + ((nb * 4ull + 7) & ~7ull);
    cudaError_t e = cudaMemsetAsync(b, 0, sb, st_);
    if (e == cudaSuccess) e = cudaMemsetAsync(c.nv, 0, 8, st_);
    if (e != cudaSuccess) return fail_cuda(e, what);
    Lookback lb;
    lb.state = reinterpret_cast<uint32_t*>(b + 16);
    lb.agg = reinterpret_cast<unsigned long long*>(b + sb);
    lb.incl = lb.agg + nb;
    launch(OB_FAM_ALIGN, ac_valid_kernel<T>, nb, kThreads, 0, st_, c.rows, c.nrm, reinterpret_cast<unsigned*>(b), lb,
           c.vp, c.vn, c.nv);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, what);
    ob_voxel_io v{};
    v.mode = c.nrm ? OB_VOXEL_POINT_NORMAL : OB_VOXEL_AVERAGE_POINT;
    v.dtype = OB_F64;
    v.points = c.vp;
    v.cols = 3;
    v.normals = c.vn;
    v.n_device = reinterpret_cast<const size_t*>(c.nv);
    v.capacity = cap;
    v.voxel_size = kVoxel;
    v.max_points_per_voxel = 1;
    v.min_pts_threshold = 1;
    v.points_out = c.fp;
    v.normals_out = c.fn;
    v.n_out = reinterpret_cast<size_t*>(c.nf);
    // AVERAGE_POINT with min_pts_threshold 1 keeps every voxel that has a row, so the reference's fallback to the
    // valid rows (an empty downsample of a non-empty cloud) cannot happen
    if (cap == 0) {
        if ((e = cudaMemsetAsync(c.nf, 0, 8, st_)) != cudaSuccess) return fail_cuda(e, what);
        return OB_OK;
    }
    return ob_voxel_downsample(&v, s_);
}

ob_status Run::wait_probe(Probe* p) {
    cudaError_t e = cudaMemcpyAsync(p, &state_->probe, sizeof(Probe), cudaMemcpyDeviceToHost, st_);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st_);
    if (e != cudaSuccess) return fail_cuda(e, "align clouds feature counts");
    return OB_OK;
}

template <bool kZ>
ob_status Run::binsum(const Cloud& c, const double* poses, unsigned groups, const BevSpec& bs, const Filter* filt,
                      uint32_t cells, double* out) {
    const size_t items = static_cast<size_t>(groups) * c.n;
    const uint32_t total = groups * cells;
    cudaError_t e = cudaMemsetAsync(out, 0, total * 8ull, st_);
    if (e != cudaSuccess) return fail_cuda(e, "align clouds grid");
    launch(OB_FAM_ALIGN, ac_items_kernel<kZ>, dim3(nblocks(c.n), groups), kThreads, 0, st_, c.fp, c.fn, c.dist,
           static_cast<unsigned>(c.n), poses, bs, filt, total, keys_, vals_, w_);
    e = sort_tmp_->run(sort_pairs(keys_, skeys_, vals_, svals_, static_cast<int>(items), 0, bits_for(total), st_));
    if (e != cudaSuccess) return fail_cuda(e, "align clouds grid sort");
    launch(OB_FAM_ALIGN, ac_segsum_kernel, nblocks(items), kThreads, 0, st_, skeys_, svals_, w_, items, total, out);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "align clouds grid");
    return OB_OK;
}

// normalise and transform one target grid; its column spectra go to tspec[col][row]
ob_status Run::target_spectrum(const Cloud& tgt, const Spec& sp, const Filter* filt, double* grid, double2* tspec,
                               int* tvalid) {
    const FftShape f = shape_of(sp);
    const BevSpec bs{sp.bound, 1.0 / sp.pixel, sp.base_n};
    ob_status rs = binsum<false>(tgt, nullptr, 1, bs, filt, f.bn * f.bn, grid);
    if (rs != OB_OK) return rs;
    const size_t smem = 2ull * f.n * sizeof(double);
    launch(OB_FAM_ALIGN, ac_norm_kernel, 1, kThreads, 0, st_, grid, f.bn * f.bn, mean_, rn_, tvalid);
    launch(OB_FAM_ALIGN, ac_fft_rows_kernel, dim3(f.bn, 1), kThreads, smem, st_, grid, f, mean_, rn_, tw_, spec_);
    launch(OB_FAM_ALIGN, ac_fft_cols_kernel<true>, dim3(f.n, 1), kThreads, smem, st_, spec_, f, tw_, nullptr, tspec);
    if (cudaError_t e = cudaGetLastError()) return fail_cuda(e, "align clouds target");
    return OB_OK;
}

// candidates first .. first + count - 1 (poses in state_->cand) against one target spectrum
ob_status Run::correlate(const Cloud& src, const Spec& sp, const double2* tspec, const int* tvalid, int first,
                         unsigned count, const Filter* filt) {
    const FftShape f = shape_of(sp);
    const unsigned W = 2 * f.ms + 1, cells = f.bn * f.bn;
    const BevSpec bs{sp.bound, 1.0 / sp.pixel, sp.base_n};
    ob_status rs = binsum<false>(src, state_->cand[first], count, bs, filt, cells, grids_);
    if (rs != OB_OK) return rs;
    const size_t smem = 2ull * f.n * sizeof(double);
    launch(OB_FAM_ALIGN, ac_norm_kernel, count, kThreads, 0, st_, grids_, cells, mean_, rn_, valid_);
    launch(OB_FAM_ALIGN, ac_fft_rows_kernel, dim3(f.bn, count), kThreads, smem, st_, grids_, f, mean_, rn_, tw_, spec_);
    launch(OB_FAM_ALIGN, ac_fft_cols_kernel<false>, dim3(f.n, count), kThreads, smem, st_, spec_, f, tw_, tspec, rows_);
    launch(OB_FAM_ALIGN, ac_fft_window_kernel, dim3(W, count), kThreads, smem, st_, rows_, f, tw_, win_);
    launch(OB_FAM_ALIGN, ac_argmax_kernel, count, kThreads, 0, st_, win_, f.ms, valid_, tvalid, first, state_);
    if (cudaError_t e = cudaGetLastError()) return fail_cuda(e, "align clouds correlation");
    return OB_OK;
}

// xy_matching_confidence at pose P (device), both directions; which: 0 initial, 1 refined
ob_status Run::confidence(Cloud& src, Cloud& tgt, bool normals, int which, const double* P) {
    Cloud* cl[2] = {&src, &tgt};
    const double cos_gate = std::cos(5.0 * kPi / 180.0);
    for (int dir = 0; dir < 2; ++dir) {
        Cloud& q = *cl[dir];
        Cloud& g = *cl[1 - dir];
        double* qr = query_[dir];
        int32_t* nn = nn_[dir];
        launch(OB_FAM_ALIGN, ac_query_kernel, nblocks(q.cap), kThreads, 0, st_, q.fp, q.nf, q.cap, P, dir, qr);
        ob_cloud_nearest_io ni{};
        ni.target = ob_point_rows{OB_F64, flat_[1 - dir], 0, reinterpret_cast<const size_t*>(g.nf), g.cap};
        ni.queries = ob_point_rows{OB_F64, qr, 0, reinterpret_cast<const size_t*>(q.nf), q.cap};
        ni.cell_size = 0.5;
        ni.max_dist_sq = 0.5 * 0.5;
        ni.indices = nn;
        ob_status rs = ob_cloud_nearest(&ni, s_);
        if (rs != OB_OK) return rs;
        launch(OB_FAM_ALIGN, ac_count_kernel, nblocks(q.cap), kThreads, 0, st_, normals ? q.fn : nullptr, q.nf, q.cap,
               mask_[dir], nn, g.fn, P, dir, cos_gate, state_->counts[which] + 2 * dir);
        if (cudaError_t e = cudaGetLastError()) return fail_cuda(e, "align clouds confidence");
    }
    return OB_OK;
}

// CUDA events at the stage boundaries of a traced call: features, pass 1 (with the target's grids and the Z shift),
// pass 2, ICP, confidence
struct StageEvents {
    cudaEvent_t ev[6] = {};
    bool on = false;
    explicit StageEvents(bool want) {
        if (!want) return;
        on = true;
        for (auto& e : ev) on = on && cudaEventCreate(&e) == cudaSuccess;
    }
    ~StageEvents() {
        for (auto e : ev)
            if (e) cudaEventDestroy(e);
    }
    void mark(int i, cudaStream_t st) {
        if (on) cudaEventRecord(ev[i], st);
    }
    void read(double* ms) const {  // after the stream is synchronised
        for (int i = 0; on && i < 5; ++i) {
            float f = 0.0f;
            if (cudaEventElapsedTime(&f, ev[i], ev[i + 1]) == cudaSuccess) ms[i] = f;
        }
    }
};

template <typename T>
ob_status run_align_clouds(Run& r, Cloud& src, Cloud& tgt, const double* guess, double* pose, double* conf,
                           std::vector<double>* fine_grid, std::vector<double>* coarse_grid, std::vector<double>* zh,
                           ob_align_clouds_trace* trace, StageEvents& ev) {
    Staging& stg = r.stg_;
    cudaStream_t st = r.st_;
    ev.mark(0, st);
    r.state_ = stg.scratch<State>(1);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "align clouds state");
    if (cudaError_t e = cudaMemsetAsync(r.state_, 0, sizeof(State), st)) return fail_cuda(e, "align clouds state");
    ob_status rs = r.features<T>(src, "align clouds source features");
    if (rs == OB_OK) rs = r.features<T>(tgt, "align clouds target features");
    if (rs != OB_OK) return rs;
    // footprint and z keys, sorted
    Cloud* cl[2] = {&src, &tgt};
    unsigned long long *ek[2], *zk[2], *eks[2], *zks[2];
    for (int c = 0; c < 2; ++c) {
        const unsigned cap = std::max(cl[c]->cap, 1u);
        ek[c] = stg.scratch<unsigned long long>(cap);
        zk[c] = stg.scratch<unsigned long long>(cap);
        eks[c] = stg.scratch<unsigned long long>(cap);
        zks[c] = stg.scratch<unsigned long long>(cap);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "align clouds keys");
        launch(OB_FAM_ALIGN, ac_keys_kernel, nblocks(cap), kThreads, 0, st, cl[c]->fp, cl[c]->nf, cl[c]->cap,
               cl[c]->dist, ek[c], zk[c]);
        const int n = static_cast<int>(cl[c]->cap);
        if (n > 0) {
            cudaError_t e = cub_run(stg, sort_keys(ek[c], eks[c], n, 0, 64, st));
            if (e == cudaSuccess) e = cub_run(stg, sort_keys(zk[c], zks[c], n, 0, 64, st));
            if (e != cudaSuccess) return fail_cuda(e, "align clouds percentile sort");
        }
    }
    launch(OB_FAM_ALIGN, ac_stats_kernel, 1, 1, 0, st, src.nf, tgt.nf, eks[0], eks[1], zks[0], zks[1], guess, r.state_);
    if (cudaError_t e = cudaGetLastError()) return fail_cuda(e, "align clouds statistics");
    ev.mark(1, st);
    Probe pr;
    if ((rs = r.wait_probe(&pr)) != OB_OK) return rs;
    src.n = pr.nf[0];
    tgt.n = pr.nf[1];
    if (trace) {
        trace->source_features = src.n;
        trace->target_features = tgt.n;
    }
    if (src.n < kMinPoints || tgt.n < kMinPoints) {  // the guess back, confidence 0
        cudaError_t e = cudaMemcpyAsync(pose, r.state_->probe.guess, 128, cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess && conf) e = cudaMemsetAsync(conf, 0, 8, st);
        if (e != cudaSuccess) return fail_cuda(e, "align clouds result");
        return OB_OK;
    }
    // project_pose_to_yaw_translation and choose_xy_matcher_params, as the oracle evaluates them
    const double* gs = pr.guess;
    double G[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    const double yaw0 = std::atan2(gs[4], gs[0]), c0 = std::cos(yaw0), s0 = std::sin(yaw0);
    G[0] = c0, G[1] = -s0, G[4] = s0, G[5] = c0;
    G[3] = gs[3], G[7] = gs[7], G[11] = gs[11];
    const double foot = std::max(pr.foot[1], pr.foot[0]);
    const double bound = std::max(10.0, std::min(60.0, std::max(foot, std::max(std::fabs(G[3]), std::fabs(G[7]))) + 2.0));
    const double max_shift_m = std::max(4.0, bound);
    const double fine_pixel = bound <= 18.0 ? 0.20 : (bound <= 30.0 ? 0.15 : 0.25);
    const Spec fine = make_spec(fine_pixel, bound, max_shift_m), coarse = make_spec(kCoarsePixel, bound, max_shift_m);
    if ((rs = r.workspace(src, tgt, fine, coarse)) != OB_OK) return rs;
    const double* dG = stg.in(G, 16);
    const double* dyaw = stg.in(yaw_table(), 16 * (kCoarseYaws + kCoarseYaws * kFineYaws));
    const bool normals = src.nrm != nullptr && tgt.nrm != nullptr;
    // target: Z histogram and both spectra
    State* S = r.state_;
    auto* zh_t = stg.scratch<double>(kZBins);
    auto* zh_m = stg.scratch<double>(kZBins);
    auto* grid_f = stg.scratch<double>(static_cast<size_t>(fine.base_n) * fine.base_n);
    auto* grid_c = stg.scratch<double>(static_cast<size_t>(coarse.base_n) * coarse.base_n);
    auto* ts_f = stg.scratch<double2>(static_cast<size_t>(fine.fft_n) * fine.fft_n);
    auto* ts_c = stg.scratch<double2>(static_cast<size_t>(coarse.fft_n) * coarse.fft_n);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "align clouds target");
    const BevSpec none{0.0, 0.0, 0};
    if ((rs = r.binsum<true>(tgt, nullptr, 1, none, nullptr, kZBins, zh_t)) != OB_OK) return rs;
    if ((rs = r.target_spectrum(tgt, fine, &S->filt_t, grid_f, ts_f, &S->target_valid[0])) != OB_OK) return rs;
    if ((rs = r.target_spectrum(tgt, coarse, &S->filt_t, grid_c, ts_c, &S->target_valid[1])) != OB_OK) return rs;
    // the Z shift, the same for every candidate (the source at G)
    if ((rs = r.binsum<true>(src, dG, 1, none, nullptr, kZBins, zh_m)) != OB_OK) return rs;
    launch(OB_FAM_ALIGN, ac_zshift_kernel, 1, kThreads, 0, st, zh_m, zh_t, r.tw_, G[11], S);
    // pass 1
    for (int first = 0; first < kCoarseYaws; first += kGroup) {
        launch(OB_FAM_ALIGN, ac_pose_kernel, 1, 32, 0, st, first, kGroup, dyaw, dG, S);
        if ((rs = r.correlate(src, coarse, ts_c, &S->target_valid[1], first, kGroup, &S->filt_s)) != OB_OK) return rs;
    }
    launch(OB_FAM_ALIGN, ac_coarse_pick_kernel, 1, 1, 0, st, S);
    ev.mark(2, st);
    // pass 2
    launch(OB_FAM_ALIGN, ac_pose_kernel, 1, 32, 0, st, -1, kFineYaws, dyaw, dG, S);
    if ((rs = r.correlate(src, fine, ts_f, &S->target_valid[0], kCoarseYaws, kFineYaws, &S->filt_s)) != OB_OK) return rs;
    launch(OB_FAM_ALIGN, ac_fine_pick_kernel, 1, 1, 0, st, dG, fine.pixel, S);
    if (cudaError_t e = cudaGetLastError()) return fail_cuda(e, "align clouds yaw search");
    ev.mark(3, st);
    // ICP
    const double gate = bound <= 18.0 ? 10.0 : 20.0;
    const double dists[3] = {2.0, 0.6, 0.25};
    for (int p = 0; p < 3; ++p) {
        ob_cloud_align_io a{};
        a.mode = normals ? OB_ALIGN_POINT_TO_PLANE : OB_ALIGN_POINT_TO_POINT;
        a.source = ob_point_rows{OB_F64, src.fp, 0, reinterpret_cast<const size_t*>(src.nf), src.cap};
        a.target = ob_point_rows{OB_F64, tgt.fp, 0, reinterpret_cast<const size_t*>(tgt.nf), tgt.cap};
        if (normals) {
            a.source_normals = src.fn;
            a.source_normal_rows = src.cap;
            a.target_normals = tgt.fn;
            a.target_normal_rows = tgt.cap;
        }
        a.initial_guess = p == 0 ? S->initial_pose : S->icp[p - 1];
        a.max_corr_dist = dists[p];
        a.max_normal_angle_deg = gate;
        a.pose = S->icp[p];
        if ((rs = ob_cloud_align(&a, r.s_)) != OB_OK) return rs;
    }
    ev.mark(4, st);
    // confidence: samples, flattened rows, the two poses
    for (int c = 0; c < 2; ++c) {
        Cloud& cc = *cl[c];
        r.flat_[c] = stg.scratch<double>(cc.cap * 3ull);
        r.mask_[c] = stg.scratch<uint8_t>(cc.cap);
        const unsigned long long* cnt = cc.nf;
        uint32_t* idx = nullptr;
        if (cc.n > kConfSamples) {
            idx = stg.scratch<uint32_t>(cc.cap);
            auto* tmp = stg.scratch<double>(cc.cap * 3ull);
            auto* sampled = stg.scratch<unsigned long long>(1);
            cnt = sampled;
            cudaError_t e = stg.error();
            if (e == cudaSuccess) e = cudaMemsetAsync(r.mask_[c], 0, cc.cap, st);
            if (e != cudaSuccess) return fail_cuda(e, "align clouds samples");
            ob_voxel_io v{};
            v.mode = OB_VOXEL_SHUFFLE_FIRST;
            v.dtype = OB_F64;
            v.points = cc.fp;
            v.cols = 3;
            v.n_device = reinterpret_cast<const size_t*>(cc.nf);
            v.capacity = cc.cap;
            v.voxel_size = kVoxel;
            v.max_points_per_voxel = 1;
            v.min_pts_threshold = 1;
            v.points_out = tmp;
            v.indices_out = idx;
            v.n_out = reinterpret_cast<size_t*>(sampled);
            if ((rs = ob_voxel_downsample(&v, r.s_)) != OB_OK) return rs;
        }
        if (cudaError_t e = stg.error()) return fail_cuda(e, "align clouds confidence");
        launch(OB_FAM_ALIGN, ac_mask_kernel, nblocks(cc.cap), kThreads, 0, st, idx, cnt, cc.cap, r.mask_[c]);
        launch(OB_FAM_ALIGN, ac_query_kernel, nblocks(cc.cap), kThreads, 0, st, cc.fp, cc.nf, cc.cap, nullptr, 0,
               r.flat_[c]);
    }
    if ((rs = r.confidence(src, tgt, normals, 0, S->initial_pose)) != OB_OK) return rs;
    if ((rs = r.confidence(src, tgt, normals, 1, S->icp[2])) != OB_OK) return rs;
    launch(OB_FAM_ALIGN, ac_finish_kernel, 1, 1, 0, st, S, r.io_->compute_confidence, pose, conf);
    ev.mark(5, st);
    if (cudaError_t e = cudaGetLastError()) return fail_cuda(e, "align clouds launch");
    if (trace) {
        trace->searched = 1;
        trace->bound_m = bound;
        trace->fine_pixel_m = fine.pixel;
        trace->coarse_pixel_m = coarse.pixel;
        trace->max_shift_m = max_shift_m;
        trace->fine_base_n = fine.base_n, trace->fine_fft_n = fine.fft_n, trace->fine_max_shift = fine.max_shift;
        trace->coarse_base_n = coarse.base_n, trace->coarse_fft_n = coarse.fft_n;
        trace->coarse_max_shift = coarse.max_shift;
        cudaError_t e = cudaSuccess;
        if (fine_grid) {
            fine_grid->resize(static_cast<size_t>(fine.base_n) * fine.base_n);
            coarse_grid->resize(static_cast<size_t>(coarse.base_n) * coarse.base_n);
            zh->resize(kZBins);
            e = cudaMemcpyAsync(fine_grid->data(), grid_f, fine_grid->size() * 8, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess)
                e = cudaMemcpyAsync(coarse_grid->data(), grid_c, coarse_grid->size() * 8, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaMemcpyAsync(zh->data(), zh_t, kZBins * 8, cudaMemcpyDeviceToHost, st);
        }
        if (e != cudaSuccess) return fail_cuda(e, "align clouds trace");
    }
    return OB_OK;
}

ob_status check_cloud(const ob_point_rows& p, size_t cols, const void* nrm, size_t nrows, size_t ncols,
                      const char* pn, const char* nn) {
    if (cols != 3) return fail(OB_INVALID_ARGUMENT, std::string(pn) + " must have shape (N, 3)");
    if (nrm || nrows || ncols) {
        if (ncols != 3) return fail(OB_INVALID_ARGUMENT, std::string(nn) + " must have shape (N, 3)");
        if (nrows != row_capacity(p.n, p.n_device, p.capacity))
            return fail(OB_INVALID_ARGUMENT, std::string(pn) + " and " + nn + " must have the same number of rows");
    }
    return OB_OK;
}

}  // namespace
}  // namespace ob

using namespace ob;

extern "C" ob_status ob_align_clouds(const ob_align_clouds_io* io, ob_stream* s) {
    if (!io || !io->pose) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = check_cloud(io->source, io->source_cols, io->source_normals, io->source_normal_rows,
                               io->source_normal_cols, "source_points", "source_normals");
    if (rs == OB_OK)
        rs = check_cloud(io->target, io->target_cols, io->target_normals, io->target_normal_rows,
                         io->target_normal_cols, "target_points", "target_normals");
    if (rs != OB_OK) return rs;
    const bool sn = io->source_normals || io->source_normal_cols, tn = io->target_normals || io->target_normal_cols;
    if (sn != tn) return fail(OB_INVALID_ARGUMENT, "source_normals and target_normals must both be given or both be omitted");
    if (io->source.dtype != io->target.dtype) return fail(OB_INVALID_ARGUMENT, "source and target must share a dtype");
    if (!s) {
        rs = require_device(0);
        return rs != OB_OK ? rs : fail(OB_INVALID_ARGUMENT, "null pointer");
    }
    const int device = stream_device(s);
    rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    Cloud src{}, tgt{};
    rs = stage_rows(&io->source, stg, &src.rows, "stage align clouds source");
    if (rs == OB_OK) rs = stage_rows(&io->target, stg, &tgt.rows, "stage align clouds target");
    if (rs != OB_OK) return rs;
    src.cap = src.rows.cap;
    tgt.cap = tgt.rows.cap;
    const size_t esz = io->source.dtype == OB_F64 ? 8 : 4;
    if (sn && ((src.cap && !io->source_normals) || (tgt.cap && !io->target_normals)))
        return fail(OB_INVALID_ARGUMENT, "null normals buffer");
    src.nrm = sn ? stg.in(io->source_normals, src.cap * 3 * esz) : nullptr;
    tgt.nrm = sn ? stg.in(io->target_normals, tgt.cap * 3 * esz) : nullptr;
    const double* guess = stg.in(io->initial_guess, 16);
    double* pose = stg.out(io->pose, 16);
    double* conf = stg.out(io->confidence, 1);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage align clouds");
    Run r(io, s, stg);
    std::vector<double> fg, cg, zh;
    ob_align_clouds_trace* tr = io->trace;
    const bool grids = tr && (tr->target_fine_grid || tr->target_coarse_grid || tr->target_z_hist);
    if (tr) {
        double *a = tr->target_fine_grid, *b = tr->target_coarse_grid, *c = tr->target_z_hist;
        std::memset(tr, 0, sizeof(*tr));
        tr->target_fine_grid = a, tr->target_coarse_grid = b, tr->target_z_hist = c;
        tr->coarse_index = tr->fine_index = -1;
    }
    StageEvents ev(tr != nullptr);
    rs = io->source.dtype == OB_F64
             ? run_align_clouds<double>(r, src, tgt, guess, pose, conf, grids ? &fg : nullptr, &cg, &zh, tr, ev)
             : run_align_clouds<float>(r, src, tgt, guess, pose, conf, grids ? &fg : nullptr, &cg, &zh, tr, ev);
    if (rs != OB_OK) return rs;
    State host{};
    const bool searched = tr && tr->searched;
    if (searched) stg.check(cudaMemcpyAsync(&host, r.state_, sizeof(State), cudaMemcpyDeviceToHost, st));
    cudaError_t e = stg.finish();
    if (e == cudaSuccess && searched) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "align clouds result");
    if (searched) {
        tr->coarse_index = host.coarse_index;
        tr->fine_index = host.fine_index;
        std::memcpy(tr->coarse_scores, host.scores, sizeof(tr->coarse_scores));
        for (int k = 0; k < kFineYaws; ++k) {
            tr->fine_z_bins[k] = host.zbins;
            tr->fine_dx[k] = host.dx[kCoarseYaws + k];
            tr->fine_dy[k] = host.dy[kCoarseYaws + k];
            tr->fine_scores[k] = host.scores[kCoarseYaws + k];
        }
        std::memcpy(tr->initial_pose, host.initial_pose, sizeof(tr->initial_pose));
        std::memcpy(tr->icp_poses, host.icp, sizeof(tr->icp_poses));
        tr->initial_confidence = host.conf[0];
        tr->refined_confidence = host.conf[1];
        tr->initial_total = host.counts[0][0] + host.counts[0][2];
        tr->initial_matched = host.counts[0][1] + host.counts[0][3];
        tr->refined_total = host.counts[1][0] + host.counts[1][2];
        tr->refined_matched = host.counts[1][1] + host.counts[1][3];
        ev.read(tr->stage_ms);
        if (grids) {
            if (tr->target_fine_grid) std::memcpy(tr->target_fine_grid, fg.data(), fg.size() * 8);
            if (tr->target_coarse_grid) std::memcpy(tr->target_coarse_grid, cg.data(), cg.size() * 8);
            if (tr->target_z_hist) std::memcpy(tr->target_z_hist, zh.data(), zh.size() * 8);
        }
    }
    return OB_OK;
}
