// ob_image.cu -- image post-processing (DESIGN f-9): AutoExposure, BeamUniformityCorrector and LocalToneMapper of
// ouster_core/src/image_processing.cpp with their state in device memory.
//
// Every arithmetic step restates the reference's in its own type with explicit rounding (__fadd_rn & co.), so
// nvcc's default contraction cannot fuse a multiply-add the reference leaves separate.  Clamps follow
// std::max / std::min argument order, so a NaN survives where the reference's does.  Order statistics come from
// a block-wide radix select on order-preserving unsigned keys; the reference's nth_element yields the same value.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "ob_api_common.h"
#include "ob_arith.cuh"

namespace ob {
namespace {

constexpr double kRLum = 0.299, kGLum = 0.587, kBLum = 0.114;
constexpr uint32_t kAeStride = 4;
constexpr uint32_t kAeMinPoints = 100;
constexpr double kBucDamping = 0.92;
constexpr int kBucEvery = 8;
constexpr int kTiles = 8;  // CLAHE_TILES_H = CLAHE_TILES_W
constexpr int kBins = 1024;
constexpr int kSelectThreads = 1024;
constexpr int kMedianThreads = 256;
constexpr int kEwThreads = 256;

// device state of one processor, and the parameter block the select step leaves for the elementwise kernels
struct DevState {
    double lo, hi, lo_state, hi_state;
    int32_t counter, initialized;
    uint32_t dc_rows;   // BUC: dark_count_.size()
    int32_t apply;      // 0: this update leaves the image as it is (early return / not initialised)
    int32_t branch;     // 0: inf/nan scale, 1: lo/hi affine, 2: hi only
    int32_t compress;   // LTM: hi_state_ < compress_dr_max_lum_
    double sub, mul, add;
};

struct HostParams {
    double lo_pct, hi_pct, damping, compress_max;
    int32_t update_every, color_correct;
};

// (r * R + g * G) + b * B in T, each constant rounded to T once
template <typename T>
__device__ __forceinline__ T lum3(T r, T g, T b) {
    return add(add(mul(r, T(kRLum)), mul(g, T(kGLum))), mul(b, T(kBLum)));
}

// f16_bits_to_f32_bits_fast_nan_zero (image_processing.cpp:59-65): a bias shift, not an IEEE conversion
__device__ __forceinline__ float f16_fast(uint16_t bits) {
    const uint32_t e = (uint32_t(bits) + 0x1C000u) << 13;
    return __uint_as_float(bits != 0 ? (bits != 0x7e00 ? e : 0u) : 0u);
}

// fast_log10 (image_processing.cpp:68-76)
__device__ __forceinline__ float fast_log10(float x) {
    const int32_t bits = __float_as_int(x);
    return __fmul_rn(__fmul_rn(__int2float_rn(bits - 0x3F800000), 1.1920929e-7f), 0.30103f);
}

// Number of items for which get(i, k) holds; every thread of the block gets the count.
template <class Get, typename K>
__device__ uint32_t block_count(const Get& get, uint32_t n_items) {
    uint32_t n = 0;
    for (uint32_t base = 0; base < n_items; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        K k;
        n += __syncthreads_count(i < n_items && get(i, k));
    }
    return n;
}

// Keys of rank rank[r] (0-based, ascending) among the items with get(i, k), for NR ranks at once: one 8-bit digit
// per pass, most significant first, each rank narrowing its own prefix.  hist: NR * 256 words of shared memory.
template <typename K, int NR, class Get>
__device__ void block_select(const Get& get, uint32_t n_items, const uint32_t* rank_in, K* out, uint32_t* hist) {
    __shared__ K prefix[NR];
    __shared__ uint32_t rank[NR];
    constexpr int kBits = int(sizeof(K) * 8);
    if (threadIdx.x < NR) {
        prefix[threadIdx.x] = 0;
        rank[threadIdx.x] = rank_in[threadIdx.x];
    }
    K hi_mask = 0;
    for (int shift = kBits - 8; shift >= 0; shift -= 8) {
        for (uint32_t i = threadIdx.x; i < NR * 256u; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        // whole warps step together, so the lanes that fall into the same bin add their count with one atomic: the
        // leading digits of similar values agree, and without this every thread would hit the same word
        const unsigned lane = threadIdx.x & 31u;
        for (uint32_t base = 0; base < n_items; base += blockDim.x) {
            const uint32_t i = base + threadIdx.x;
            K k = 0;
            const bool valid = i < n_items && get(i, k);
            const uint32_t d = uint32_t(k >> shift) & 255u;
#pragma unroll
            for (int r = 0; r < NR; ++r) {
                const bool hit = valid && (k & hi_mask) == prefix[r];
                const unsigned peers = __match_any_sync(0xffffffffu, hit ? d : 0xffffffffu);
                if (hit && lane == unsigned(__ffs(peers) - 1)) atomicAdd(&hist[r * 256 + d], unsigned(__popc(peers)));
            }
        }
        __syncthreads();
        if (threadIdx.x < NR) {
            const int r = threadIdx.x;
            uint32_t cum = 0;
            for (int b = 0; b < 256; ++b) {
                const uint32_t c = hist[r * 256 + b];
                if (rank[r] < cum + c) {
                    prefix[r] |= K(b) << shift;
                    rank[r] -= cum;
                    break;
                }
                cum += c;
            }
        }
        __syncthreads();
        hi_mask |= K(255) << shift;
    }
    if (threadIdx.x < NR) out[threadIdx.x] = prefix[threadIdx.x];
    __syncthreads();
}

// layouts: 0 mono T, 1 rgb T, 2 rgb float16 bits (T = float)
template <typename T, int L>
__device__ __forceinline__ T load(const void* p, size_t i) {
    if constexpr (L == 2) return f16_fast(static_cast<const uint16_t*>(p)[i]);
    else return static_cast<const T*>(p)[i];
}

// AutoExposure::apply / LocalToneMapper::apply up to the affine map: the candidates (every 4th pixel, value or
// luminance > 0), the two order statistics, initialisation, damping, the branch and the counter.
template <typename T, int L>
__global__ void __launch_bounds__(kSelectThreads) ae_select_kernel(const void* img, uint32_t npx, DevState* st,
                                                                    HostParams p, int update_state, int ltm) {
    using K = decltype(okey(T()));
    __shared__ uint32_t hist[2 * 256];
    __shared__ int select;
    // one read of the counter, shared before anyone branches on it: thread 0 writes it back further down
    if (threadIdx.x == 0) select = st->counter == 0 && update_state;
    __syncthreads();
    if (select) {
        const uint32_t n_items = (npx + kAeStride - 1) / kAeStride;
        auto get = [&](uint32_t i, K& k) -> bool {
            const size_t px = size_t(i) * kAeStride;
            T v;
            if constexpr (L == 0) v = load<T, L>(img, px);
            else v = lum3<T>(load<T, L>(img, 3 * px), load<T, L>(img, 3 * px + 1), load<T, L>(img, 3 * px + 2));
            if (!(v > T(0))) return false;
            k = okey(v);
            return true;
        };
        const uint32_t n = block_count<decltype(get), K>(get, n_items);
        if (n < kAeMinPoints) {  // too few nonzero values: return without touching the image or the counter
            if (threadIdx.x == 0) st->apply = 0;
            return;
        }
        const uint32_t k_lo = uint32_t(__double2ull_rz(__dmul_rn(double(n), p.lo_pct)));
        const uint32_t k_hi = uint32_t(__double2ull_rz(__dmul_rn(double(n), p.hi_pct)));
        const uint32_t ranks[2] = {k_lo, n - k_hi - 1};
        __shared__ K res[2];
        block_select<K, 2>(get, n_items, ranks, res, hist);
        if (threadIdx.x == 0) {
            st->lo = double(okey_value(res[0]));
            st->hi = double(okey_value(res[1]));
            if (!st->initialized) {
                st->initialized = 1;
                st->lo_state = st->lo;
                st->hi_state = st->hi;
            }
        }
    }
    if (threadIdx.x != 0) return;
    if (!st->initialized) {
        st->apply = 0;
        return;
    }
    double ls = st->lo_state, hs = st->hi_state;
    if (update_state) {
        const double d = p.damping, e = __dsub_rn(1.0, p.damping);
        ls = __dadd_rn(__dmul_rn(d, ls), __dmul_rn(e, st->lo));
        hs = __dadd_rn(__dmul_rn(d, hs), __dmul_rn(e, st->hi));
        st->lo_state = ls;
        st->hi_state = hs;
    }
    const double scale = __ddiv_rn(__dsub_rn(1.0, __dadd_rn(p.lo_pct, p.hi_pct)), __dsub_rn(hs, ls));
    if (isinf(scale) || isnan(scale)) {
        st->branch = 0;
        st->mul = __ddiv_rn(0.5, hs);
    } else if (__dadd_rn(__dmul_rn(scale, __dsub_rn(0.0, ls)), p.lo_pct) <= 0.0) {
        st->branch = 1;
        st->sub = ls;
        st->mul = scale;
        st->add = p.lo_pct;
    } else {
        st->branch = 2;
        st->mul = __ddiv_rn(__dsub_rn(1.0, p.hi_pct), hs);
    }
    if (update_state) st->counter = (st->counter + 1) % p.update_every;
    st->compress = ltm && (hs < p.compress_max);
    st->apply = 1;
}

template <typename T>
__device__ __forceinline__ T affine(T v, const DevState& s) {
    if (s.branch == 1) return add(mul(sub(v, T(s.sub)), T(s.mul)), T(s.add));
    return mul(v, T(s.mul));
}

// AutoExposure: the affine map and the clamp to [0, 1]; the float16 layout always writes the converted input
template <typename T, int L>
__global__ void ae_apply_kernel(const void* in, T* out, size_t n, const DevState* st) {
    const DevState s = *st;
    if (!s.apply && L != 2) return;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) {
        T v = load<T, L>(in, i);
        if (s.apply) v = smin(smax(affine(v, s), T(0)), T(1));
        out[i] = v;
    }
}

// LocalToneMapper stages 1-2 and Reinhard: affine map (no clamp), dynamic-range compression, max(0), x / (1 + x);
// writes the image and its luminance lum_ae
template <typename T, int L>
__global__ void ltm_pixel_kernel(const void* in, T* out, T* lum_ae, uint32_t npx, const DevState* st) {
    const DevState s = *st;
    if (!s.apply && L != 2) return;
    const T thresh = T(0.8);
    for (uint32_t px = blockIdx.x * blockDim.x + threadIdx.x; px < npx; px += gridDim.x * blockDim.x) {
        T c[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = load<T, L>(in, 3 * size_t(px) + k);
        if (s.apply) {
#pragma unroll
            for (int k = 0; k < 3; ++k) c[k] = affine(c[k], s);
            if (s.compress) {
                const T lum = lum3(c[0], c[1], c[2]);
                if (lum > thresh) {
                    // lum - thresh + 1.0 is a double expression, narrowed to float for fast_log10
                    const float arg = __double2float_rn(__dadd_rn(double(sub(lum, thresh)), 1.0));
                    const T new_lum = add(thresh, T(fast_log10(arg)));
                    const T scale = div(new_lum, lum);
#pragma unroll
                    for (int k = 0; k < 3; ++k) c[k] = mul(c[k], scale);
                }
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const T x = smax(c[k], T(0));
                c[k] = div(x, add(T(1), x));
            }
            lum_ae[px] = lum3(c[0], c[1], c[2]);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) out[3 * size_t(px) + k] = c[k];
    }
}

// the reference's min((int)(float(lum) * 1024), 1023); a NaN luminance, whose int cast is undefined there, goes to bin 0
template <typename T>
__device__ __forceinline__ int clahe_bin(T lum) {
    const float f = __fmul_rn(float(lum), float(kBins));
    return isnan(f) ? 0 : min(__float2int_rz(f), kBins - 1);
}

// compute_clahe_luts: one CTA per tile; integer counts in shared memory (exact as floats), then one thread runs the
// clip, the excess and the CDF in bin order, as the reference's float sums do
template <typename T>
__global__ void __launch_bounds__(1024) clahe_lut_kernel(const T* lum, int h, int w, float* luts, const DevState* st) {
    if (!st->apply) return;
    __shared__ uint32_t cnt[kBins];
    const int ty = blockIdx.x / kTiles, tx = blockIdx.x % kTiles;
    const int y0 = ty * h / kTiles, y1 = (ty + 1) * h / kTiles;
    const int x0 = tx * w / kTiles, x1 = (tx + 1) * w / kTiles;
    const int tw = x1 - x0, tile_pixels = (y1 - y0) * tw;
    for (int i = threadIdx.x; i < kBins; i += blockDim.x) cnt[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < tile_pixels; i += blockDim.x) {
        const int y = y0 + i / tw, x = x0 + i % tw;
        atomicAdd(&cnt[clahe_bin(lum[size_t(y) * w + x])], 1u);
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const float clip = __fdiv_rn(__fmul_rn(1.0f, float(tile_pixels)), float(kBins));
    float excess = 0.0f;
    for (int b = 0; b < kBins; ++b) {
        const float hb = float(cnt[b]);
        if (hb > clip) excess = __fadd_rn(excess, __fsub_rn(hb, clip));
    }
    const float redistribute = __fdiv_rn(excess, float(kBins));
    const float inv_pix = __fdiv_rn(1.0f, float(tile_pixels));
    float cdf = 0.0f;
    float* lut = luts + size_t(blockIdx.x) * kBins;
    for (int b = 0; b < kBins; ++b) {
        float hb = float(cnt[b]);
        if (hb > clip) hb = clip;
        cdf = __fadd_rn(cdf, __fadd_rn(hb, redistribute));
        lut[b] = smin(__fmul_rn(cdf, inv_pix), 1.0f);
    }
}

// (float(i) + 0.5f) * tiles / n - 0.5f, its tile and weight
__device__ __forceinline__ void tile_coord(int i, int n, int& t0, int& t1, float& f) {
    const float tf = __fsub_rn(__fdiv_rn(__fmul_rn(__fadd_rn(float(i), 0.5f), float(kTiles)), float(n)), 0.5f);
    t0 = max(0, min(kTiles - 1, int(floorf(tf))));
    t1 = min(kTiles - 1, t0 + 1);
    f = __fsub_rn(tf, float(t0));
}

// apply_clahe_luts and stages 3-4: bilinear LUT lookup, the luminance ratio and the colour stage
template <typename T>
__global__ void ltm_apply_kernel(T* img, const T* lum_ae, int h, int w, const float* luts, const DevState* st,
                                 int color_correct) {
    const DevState s = *st;
    if (!s.apply) return;
    T cf = T(0.75);
    if (s.hi_state < 1.0) cf = mul(cf, smax(T(0), T(__ddiv_rn(__dsub_rn(s.hi_state, 0.5), 0.5))));
    const bool plain = !color_correct || cf == T(0);
    const uint32_t npx = uint32_t(h) * uint32_t(w);
    for (uint32_t px = blockIdx.x * blockDim.x + threadIdx.x; px < npx; px += gridDim.x * blockDim.x) {
        const int y = int(px / uint32_t(w)), x = int(px % uint32_t(w));
        int ty0, ty1, tx0, tx1;
        float fy, fx;
        tile_coord(y, h, ty0, ty1, fy);
        tile_coord(x, w, tx0, tx1, fx);
        const T lum_old = lum_ae[px];
        const int bin = clahe_bin(lum_old);
        const float* l0 = luts + size_t(ty0) * kTiles * kBins;
        const float* l1 = luts + size_t(ty1) * kTiles * kBins;
        const float gx = __fsub_rn(1.0f, fx);
        const float a = __fadd_rn(__fmul_rn(gx, l0[tx0 * kBins + bin]), __fmul_rn(fx, l0[tx1 * kBins + bin]));
        const float b = __fadd_rn(__fmul_rn(gx, l1[tx0 * kBins + bin]), __fmul_rn(fx, l1[tx1 * kBins + bin]));
        const T lum_new = T(__fadd_rn(__fmul_rn(__fsub_rn(1.0f, fy), a), __fmul_rn(fy, b)));
        const T scale = (lum_old > T(1e-6)) ? div(lum_new, lum_old) : T(1);
        T* c = img + 3 * size_t(px);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const T v = mul(c[k], scale);
            if (plain) {
                c[k] = smin(v, T(1));
            } else {
                const T u = add(mul(-lum_new, cf), mul(v, add(T(1), cf)));
                c[k] = smax(T(0), smin(u, T(1)));
            }
        }
    }
}

// ---- BeamUniformityCorrector ----
__device__ __forceinline__ bool buc_recompute(const DevState* st, uint32_t rows, int update_state) {
    return st->dc_rows != rows || (update_state && st->counter == 0);
}

// col_mask = image.cast<bool>().colwise().any()
template <typename T>
__global__ void buc_mask_kernel(const T* img, uint32_t rows, uint32_t cols, uint8_t* mask, const DevState* st,
                                int update_state) {
    if (!buc_recompute(st, rows, update_state)) return;
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += gridDim.x * blockDim.x) {
        uint8_t any = 0;
        for (uint32_t r = 0; r < rows && !any; ++r) any = img[size_t(r) * cols + c] != T(0);
        mask[c] = any;
    }
}

// element n_cols / 2 of the masked differences of rows (i, i - 1), i = blockIdx.x + 1
template <typename T>
__global__ void __launch_bounds__(kMedianThreads) buc_median_kernel(const T* img, uint32_t rows, uint32_t cols,
                                                                     const uint8_t* mask, T* med, const DevState* st,
                                                                     int update_state) {
    using K = decltype(okey(T()));
    if (!buc_recompute(st, rows, update_state)) return;
    __shared__ uint32_t hist[256];
    __shared__ K res;
    const uint32_t i = blockIdx.x + 1;
    const T* a = img + size_t(i) * cols;
    const T* b = a - cols;
    auto get = [&](uint32_t c, K& k) -> bool {
        if (!mask[c]) return false;
        k = okey(sub(a[c], b[c]));
        return true;
    };
    const uint32_t n = block_count<decltype(get), K>(get, cols);
    if (n == 0) return;
    const uint32_t rank = n / 2;
    block_select<K, 1>(get, cols, &rank, &res, hist);
    if (threadIdx.x == 0) med[i] = okey_value(res);
}

// compute_dark_count after the medians: the cumulative sum, the FullPivLU "fit" (restated below), the minimum, then
// the damping in double; one thread.  Also advances the counter, which BUC does on every call.
template <typename T>
__global__ void buc_tail_kernel(uint32_t rows, uint32_t cols, const uint8_t* mask, T* dc, T* lu, double* dark,
                                DevState* st, int update_state) {
    const bool reset = st->dc_rows != rows;
    if (reset || (update_state && st->counter == 0)) {
        uint32_t n_cols = 0;
        for (uint32_t c = 0; c < cols; ++c) n_cols += mask[c];
        const int h = int(rows);
        if (n_cols == 0) {
            for (int i = 0; i < h; ++i) dc[i] = T(0);
        } else {
            dc[0] = T(0);
            for (int i = 1; i < h; ++i) dc[i] = add(dc[i - 1], dc[i]);  // dc[i] held the median of pair i
            // image_array.fullPivLu().solve(dc) for image_array = [1, i] (h x 2), lu column-major
            T* c0 = lu;
            T* c1 = lu + h;
            T* cv = lu + 2 * h;
            for (int i = 0; i < h; ++i) {
                c0[i] = T(1);
                c1[i] = T(i);
            }
            T* col[2] = {c0, c1};
            const int size = min(h, 2);
            int rowt[2] = {0, 1}, colt[2] = {0, 1};
            int nonzero = size;
            T maxpivot = T(0);
            for (int k = 0; k < size; ++k) {
                // maxCoeff of |bottomRightCorner|: first strict maximum in column-major order
                int br = k, bc = k;
                T best = fabs(col[k][k]);
                for (int j = k; j < 2; ++j)
                    for (int r = (j == k ? k + 1 : k); r < h; ++r)
                        if (fabs(col[j][r]) > best) {
                            best = fabs(col[j][r]);
                            br = r;
                            bc = j;
                        }
                if (best == T(0)) {
                    nonzero = k;
                    for (int q = k; q < size; ++q) rowt[q] = colt[q] = q;
                    break;
                }
                if (best > maxpivot) maxpivot = best;
                rowt[k] = br;
                colt[k] = bc;
                if (br != k)
                    for (int j = 0; j < 2; ++j) {
                        const T t = col[j][k];
                        col[j][k] = col[j][br];
                        col[j][br] = t;
                    }
                if (bc != k) {
                    T* t = col[k];
                    col[k] = col[bc];
                    col[bc] = t;
                }
                for (int r = k + 1; r < h; ++r) col[k][r] = div(col[k][r], col[k][k]);
                if (k < size - 1)
                    for (int j = k + 1; j < 2; ++j)
                        for (int r = k + 1; r < h; ++r) col[j][r] = sub(col[j][r], mul(col[k][r], col[j][k]));
            }
            const T thr = mul(maxpivot, mul(T(sizeof(T) == 4 ? 1.1920928955078125e-07 : 2.220446049250313e-16),
                                              T(size)));
            int rank = 0;
            for (int q = 0; q < nonzero; ++q) rank += fabs(col[q][q]) > thr;
            T x[2] = {T(0), T(0)};
            if (rank > 0) {
                // c = P * rhs: the row transpositions applied in order
                for (int i = 0; i < h; ++i) cv[i] = dc[i];
                for (int k = 0; k < size; ++k) {
                    const T t = cv[k];
                    cv[k] = cv[rowt[k]];
                    cv[rowt[k]] = t;
                }
                T c[2] = {cv[0], size > 1 ? cv[1] : T(0)};
                if (size > 1) c[1] = sub(c[1], mul(c[0], col[0][1]));  // unit lower
                // upper, rank x rank, back substitution
                if (rank > 1) {
                    c[1] = div(c[1], col[1][1]);
                    c[0] = sub(c[0], mul(c[1], col[1][0]));
                }
                c[0] = div(c[0], col[0][0]);
                int q[2] = {0, 1};
                for (int k = 0; k < size; ++k) {
                    const int t = colt[k], s = q[k];
                    q[k] = q[t];
                    q[t] = s;
                }
                for (int k = 0; k < rank; ++k) x[q[k]] = c[k];
            }
            T m = T(0);
            for (int i = 0; i < h; ++i) {
                dc[i] = sub(dc[i], add(mul(T(1), x[0]), mul(T(i), x[1])));
                m = (i == 0) ? dc[i] : smin(m, dc[i]);
            }
            for (int i = 0; i < h; ++i) dc[i] = sub(dc[i], m);
        }
        for (int i = 0; i < h; ++i)
            dark[i] = reset ? double(dc[i])
                            : __dadd_rn(__dmul_rn(dark[i], kBucDamping), __dmul_rn(double(dc[i]), 1.0 - kBucDamping));
        st->dc_rows = rows;
    }
    st->counter = (st->counter + 1) % kBucEvery;
}

// image.colwise() -= dark_count_.cast<T>(); image = image.cwiseMax(0)
template <typename T>
__global__ void buc_apply_kernel(T* img, uint32_t cols, size_t n, const double* dark) {
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x)
        img[i] = smax(sub(img[i], T(dark[i / cols])), T(0));
}

unsigned ew_blocks(size_t n) { return unsigned(std::max<size_t>(1, std::min<size_t>((n + kEwThreads - 1) / kEwThreads, 4096))); }

}  // namespace
}  // namespace ob

struct ob_image_proc {
    int device, kind;
    ob::HostParams p;
    ob::DeviceBlock st;       // one DevState
    ob::DeviceBlock scratch;  // per-update scratch of BUC and LTM
    ob::DeviceBlock dark;     // BUC's dark count, double x rows
};

using namespace ob;

namespace {

template <typename T, int L>
void launch_ae(ob_image_proc* p, const void* in, T* out, uint32_t npx, int update_state, cudaStream_t st) {
    DevState* ds = p->st.get<DevState>();
    launch(OB_FAM_IMAGE, ae_select_kernel<T, L>, 1, kSelectThreads, 0, st, in, npx, ds, p->p, update_state, 0);
    const size_t n = size_t(npx) * (L == 0 ? 1 : 3);
    launch(OB_FAM_IMAGE, ae_apply_kernel<T, L>, ew_blocks(n), kEwThreads, 0, st, in, out, n, ds);
}

template <typename T, int L>
void launch_ltm(ob_image_proc* p, const void* in, T* out, uint32_t rows, uint32_t cols, int update_state,
                cudaStream_t st) {
    const uint32_t npx = rows * cols;
    DevState* ds = p->st.get<DevState>();
    T* lum = p->scratch.get<T>();
    float* luts = reinterpret_cast<float*>(p->scratch.get<char>() + ((size_t(npx) * sizeof(T) + 255) & ~size_t(255)));
    launch(OB_FAM_IMAGE, ae_select_kernel<T, L>, 1, kSelectThreads, 0, st, in, npx, ds, p->p, update_state, 1);
    launch(OB_FAM_IMAGE, ltm_pixel_kernel<T, L>, ew_blocks(npx), kEwThreads, 0, st, in, out, lum, npx, ds);
    launch(OB_FAM_IMAGE, clahe_lut_kernel<T>, kTiles * kTiles, 1024, 0, st, lum, int(rows), int(cols), luts, ds);
    launch(OB_FAM_IMAGE, ltm_apply_kernel<T>, ew_blocks(npx), kEwThreads, 0, st, out, lum, int(rows), int(cols), luts,
           ds, p->p.color_correct);
}

template <typename T>
void launch_buc(ob_image_proc* p, T* img, uint32_t rows, uint32_t cols, int update_state, cudaStream_t st) {
    DevState* ds = p->st.get<DevState>();
    double* dark = p->dark.get<double>();
    uint8_t* mask = p->scratch.get<uint8_t>();
    T* dc = reinterpret_cast<T*>(p->scratch.get<char>() + ((size_t(cols) + 255) & ~size_t(255)));
    T* lu = dc + rows;
    launch(OB_FAM_IMAGE, buc_mask_kernel<T>, ew_blocks(cols), kEwThreads, 0, st, img, rows, cols, mask, ds,
           update_state);
    if (rows > 1)
        launch(OB_FAM_IMAGE, buc_median_kernel<T>, rows - 1, kMedianThreads, 0, st, img, rows, cols, mask, dc, ds,
               update_state);
    launch(OB_FAM_IMAGE, buc_tail_kernel<T>, 1, 1, 0, st, rows, cols, mask, dc, lu, dark, ds, update_state);
    const size_t n = size_t(rows) * cols;
    launch(OB_FAM_IMAGE, buc_apply_kernel<T>, ew_blocks(n), kEwThreads, 0, st, img, cols, n, dark);
}

}  // namespace

extern "C" {

ob_status ob_image_proc_create(int device, int kind, const ob_image_params* params, ob_image_proc** out) {
    if (!out) return fail(OB_INVALID_ARGUMENT, "null pointer");
    *out = nullptr;
    if (kind < OB_IMAGE_AUTO_EXPOSURE || kind > OB_IMAGE_LOCAL_TONE_MAP) return fail(OB_INVALID_ARGUMENT, "unknown kind");
    HostParams hp{0, 0, 0, 0, 1, 0};
    if (kind != OB_IMAGE_BEAM_UNIFORMITY) {
        if (!params) return fail(OB_INVALID_ARGUMENT, "null pointer");
        if (!(params->lo_percentile >= 0.0 && params->lo_percentile < 1.0) ||
            !(params->hi_percentile >= 0.0 && params->hi_percentile < 1.0))
            return fail(OB_INVALID_ARGUMENT, "lo_percentile and hi_percentile must be in [0, 1)");
        if (params->update_every < 1) return fail(OB_INVALID_ARGUMENT, "update_every must be >= 1");
        hp = HostParams{params->lo_percentile, params->hi_percentile, params->damping, params->compress_dr_max_lum,
                        params->update_every, params->color_correct};
    }
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    std::unique_ptr<ob_image_proc> p(new ob_image_proc{device, kind, hp});
    cudaError_t e = p->st.alloc(sizeof(DevState));
    DevState s0{};
    s0.lo = s0.hi = s0.lo_state = s0.hi_state = -1.0;
    if (e == cudaSuccess) e = cudaMemcpy(p->st.get(), &s0, sizeof(s0), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return fail_cuda(e, "ob_image_proc_create");
    *out = p.release();
    return OB_OK;
}

ob_status ob_image_proc_update(ob_image_proc* p, int layout, int dtype, const void* in, void* out, uint32_t rows,
                               uint32_t cols, int update_state, ob_stream* s) {
    if (!p || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const bool f16 = layout == OB_IMAGE_RGB_F16;
    const bool ok_layout = (layout == OB_IMAGE_MONO && p->kind != OB_IMAGE_LOCAL_TONE_MAP) ||
                           ((layout == OB_IMAGE_RGB || f16) && p->kind != OB_IMAGE_BEAM_UNIFORMITY);
    if (!ok_layout || (dtype != OB_F32 && dtype != OB_F64) || (f16 && dtype != OB_F32))
        return fail(OB_INVALID_ARGUMENT, "layout not supported by this processor");
    const size_t npx = size_t(rows) * cols;
    const size_t n = npx * (layout == OB_IMAGE_MONO ? 1 : 3);
    if (n > 0x7fffffffull) return fail(OB_INVALID_ARGUMENT, "image too large");
    if (p->kind == OB_IMAGE_BEAM_UNIFORMITY && npx == 0) return fail(OB_INVALID_ARGUMENT, "empty image");
    if (n && (!out || (f16 && !in))) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (!f16 && in && in != out) return fail(OB_INVALID_ARGUMENT, "the image is updated in place: in must be NULL or out");
    if (stream_device(s) != p->device)
        return fail(OB_INVALID_ARGUMENT, "stream and processor are on different devices");
    ob_status rs = require_device(p->device);
    if (rs != OB_OK) return rs;
    if (n == 0) return OB_OK;  // no candidates: AE and LTM return early
    cudaStream_t st = stream_handle(s);
    const size_t esz = dtype == OB_F64 ? 8 : 4;
    cudaError_t e = cudaSuccess;
    if (p->kind == OB_IMAGE_BEAM_UNIFORMITY) {
        e = p->scratch.reserve(((size_t(cols) + 255) & ~size_t(255)) + 4 * size_t(rows) * esz);
        // the dark count keeps its values across calls only while the height stays the same; a new height
        // recomputes it, so a larger buffer need not carry the old one over
        if (e == cudaSuccess) e = p->dark.reserve(size_t(rows) * 8);
    } else if (p->kind == OB_IMAGE_LOCAL_TONE_MAP) {
        e = p->scratch.reserve(((npx * esz + 255) & ~size_t(255)) + size_t(kTiles * kTiles * kBins) * 4);
    }
    if (e != cudaSuccess) return fail_cuda(e, "image scratch");
    Staging stg(st);
    const void* din = nullptr;
    void* dout = nullptr;
    if (f16) {
        din = stg.in(in, n * 2);
        dout = stg.out(out, n * 4);
    } else {
        din = dout = stg.inout(out, n * esz);
    }
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage image");
    const uint32_t np = uint32_t(npx);
    const int us = update_state ? 1 : 0;
    if (p->kind == OB_IMAGE_AUTO_EXPOSURE) {
        if (f16) launch_ae<float, 2>(p, din, static_cast<float*>(dout), np, us, st);
        else if (layout == OB_IMAGE_MONO && dtype == OB_F32) launch_ae<float, 0>(p, din, static_cast<float*>(dout), np, us, st);
        else if (layout == OB_IMAGE_MONO) launch_ae<double, 0>(p, din, static_cast<double*>(dout), np, us, st);
        else if (dtype == OB_F32) launch_ae<float, 1>(p, din, static_cast<float*>(dout), np, us, st);
        else launch_ae<double, 1>(p, din, static_cast<double*>(dout), np, us, st);
    } else if (p->kind == OB_IMAGE_LOCAL_TONE_MAP) {
        if (f16) launch_ltm<float, 2>(p, din, static_cast<float*>(dout), rows, cols, us, st);
        else if (dtype == OB_F32) launch_ltm<float, 1>(p, din, static_cast<float*>(dout), rows, cols, us, st);
        else launch_ltm<double, 1>(p, din, static_cast<double*>(dout), rows, cols, us, st);
    } else {
        if (dtype == OB_F32) launch_buc<float>(p, static_cast<float*>(dout), rows, cols, us, st);
        else launch_buc<double>(p, static_cast<double*>(dout), rows, cols, us, st);
    }
    stg.check(cudaGetLastError());
    e = stg.flush();
    if (e == cudaSuccess && (!is_device_ptr(out) || (f16 && !is_device_ptr(in)))) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "image update");
    return OB_OK;
}

ob_status ob_image_proc_state(const ob_image_proc* p, ob_image_state* state, double* dark_count, size_t cap,
                              ob_stream* s) {
    if (!p || !state || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (stream_device(s) != p->device)
        return fail(OB_INVALID_ARGUMENT, "stream and processor are on different devices");
    ob_status rs = require_device(p->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    DevState d;
    cudaError_t e = cudaMemcpyAsync(&d, p->st.get(), sizeof(d), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    size_t nd = 0;
    if (e == cudaSuccess && dark_count && p->dark.get()) {
        nd = std::min<size_t>(d.dc_rows, cap);
        if (nd) e = cudaMemcpyAsync(dark_count, p->dark.get(), nd * 8, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e != cudaSuccess) return fail_cuda(e, "image state");
    *state = ob_image_state{d.lo, d.hi, d.lo_state, d.hi_state, d.counter, d.initialized, d.dc_rows, 0};
    return OB_OK;
}

ob_status ob_image_proc_destroy(ob_image_proc* p) {
    if (!p) return OB_OK;
    DeviceScope on(p->device);
    delete p;
    return OB_OK;
}

}  // extern "C"
