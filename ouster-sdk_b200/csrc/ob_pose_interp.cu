// ob_pose_interp.cu -- pose interpolation (DESIGN f-12): core::interp_pose / interp_pose_float and the
// constant-velocity deskew of a FrameSet.
//
// What it replaces (reference paths relative to the reference tree):
//   impl::interp_pose_range (two-pose form)         ouster_core/include/ouster/core/pose_util.h:194-235
//   impl::interp_pose (knot form)                   pose_util.h:243-286
//   interp_pose overloads                           pose_util.h:316-434
//   mapping::impl::interp_pose(frame, t0, x0, t1, x1), ConstantVelocityDeskewMethod::update
//                                                   ouster_mapping/src/deskew_method.cpp:29-37, 55-71
//   impl::init_valid_column_poses                   ouster_mapping/src/slam_util.cpp:129-140
//
// ob_interp_pose, three launches (one when n == 0):
//   scan    grid over x: the first strict descent x[j] < x[j-1] and whether x holds a NaN;
//   plan    one block: the reference's partition of x into segments and its first error.  For x without NaN and
//           without a descent, lower_bound from the previous boundary equals the running maximum of independent
//           lower_bounds from the start, so every knot is searched in parallel.  Otherwise thread 0 walks the knots
//           exactly as the reference does (libstdc++'s lower_bound on the unsorted x).  A descent anywhere fails the
//           call: a boundary never separates one (lower_bound leaves x[it-1] < knot <= x[it]), so the first descent
//           is reported in the range that holds it, unless a knot check or a zero duration comes first.  Each
//           segment's scaled twist log(a^-1 b) / duration is computed here once;
//   interp  one thread per query: its segment, dt, exp, a * exp, rounded once to the pose dtype; the block's rows
//           are staged in shared memory and leave as contiguous 16-byte stores.  Nothing is written on an error.
// ob_frames_interp_pose, two launches (one for the constant pose): a check block per frame finds the first descent
// of its valid timestamps; the write kernel then poses the valid columns of the frames before the first failing one.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "ob_api_common.h"
#include "ob_se3.cuh"

namespace ob {
namespace {

constexpr unsigned kPlanThreads = 256;
constexpr unsigned kQThreads = 128;  // queries per interp block
constexpr unsigned kCheckThreads = 256;
constexpr unsigned kWriteThreads = 128;
constexpr unsigned long long kNone = ~0ull;

struct Seg {  // one knot segment: a, the scaled twist, t0 (raw 8 bytes of the x dtype)
    double a[16];
    double tw[6];
    long long t0;
};

struct ScanFlags {
    unsigned long long first_desc;  // kNone: no descent
    unsigned nan;
    unsigned pad;
};

template <typename T>
__device__ __forceinline__ long long raw(T v) {
    long long r;
    memcpy(&r, &v, 8);
    return r;
}
template <typename T>
__device__ __forceinline__ T from_raw(long long r) {
    T v;
    memcpy(&v, &r, 8);
    return v;
}
// std::numeric_limits<T>::epsilon(): 0 for int64, so an int64 duration is never too short
template <typename T>
__device__ __forceinline__ bool zero_duration(T t0, T t1);
template <>
__device__ __forceinline__ bool zero_duration<double>(double t0, double t1) { return fabs(t1 - t0) < DBL_EPSILON; }
template <>
__device__ __forceinline__ bool zero_duration<long long>(long long, long long) { return false; }

__global__ void __launch_bounds__(256) scan_kernel_f64(const double* x, size_t n, ScanFlags* fl) {
    unsigned long long first = kNone;
    bool nan = false;
    for (size_t j = blockIdx.x * 256ull + threadIdx.x; j < n; j += static_cast<size_t>(gridDim.x) * 256) {
        const double v = x[j];
        nan |= v != v;
        if (j > 0 && first == kNone && v < x[j - 1]) first = j;
    }
    if (first != kNone) atomicMin(&fl->first_desc, first);
    if (nan) atomicOr(&fl->nan, 1u);
}
__global__ void __launch_bounds__(256) scan_kernel_i64(const long long* x, size_t n, ScanFlags* fl) {
    unsigned long long first = kNone;
    for (size_t j = blockIdx.x * 256ull + threadIdx.x; j < n; j += static_cast<size_t>(gridDim.x) * 256)
        if (j > 0 && first == kNone && x[j] < x[j - 1]) first = j;
    if (first != kNone) atomicMin(&fl->first_desc, first);
}

// std::lower_bound as libstdc++ runs it (any input order)
template <typename T>
__device__ size_t lower_bound_walk(const T* x, size_t first, size_t last, T val) {
    size_t len = last - first;
    while (len > 0) {
        const size_t half = len >> 1;
        const size_t mid = first + half;
        if (x[mid] < val) {
            first = mid + 1;
            len = len - half - 1;
        } else {
            len = half;
        }
    }
    return first;
}

template <typename P>
__device__ __forceinline__ double widen(const P* p, size_t i) { return static_cast<double>(p[i]); }

// segment i: a = poses[i], b = poses[i + 1], twist = log(a^-1 b) * (1 / (t1 - t0)) with the duration in T
template <typename T, typename P>
__device__ void make_seg(const T* knots, const P* poses, size_t i, Seg* s) {
    double a[16], b[16], ai[16], r[16], tw[6];
    for (int k = 0; k < 16; ++k) {
        a[k] = widen(poses, 16 * i + k);
        b[k] = widen(poses, 16 * (i + 1) + k);
    }
    inverse4(a, ai);
    mat4_mul(ai, b, r);
    poseh_log(r, tw);
    const T duration = knots[i + 1] - knots[i];
    const double inv = 1.0 / static_cast<double>(duration);
    for (int k = 0; k < 16; ++k) s->a[k] = a[k];
    for (int k = 0; k < 6; ++k) s->tw[k] = mul(inv, tw[k]);
    s->t0 = raw(knots[i]);
}

// error words: kind, index, frame; vals (internal, nullable): raw bits of x[index], x[index - 1]
__device__ void put_error(long long* err, long long* vals, int kind, long long index, long long frame, long long cur,
                          long long prev) {
    err[0] = kind;
    err[1] = index;
    err[2] = frame;
    if (vals) {
        vals[0] = cur;
        vals[1] = prev;
    }
}

template <typename T, typename P>
__global__ void __launch_bounds__(kPlanThreads) plan_kernel(const T* x, size_t n, const T* knots, size_t m, const P* poses,
                                                            int two_pose, const ScanFlags* fl, size_t* ends, Seg* segs,
                                                            long long* err, long long* vals) {
    using BS = cub::BlockScan<unsigned long long, kPlanThreads>;
    __shared__ typename BS::TempStorage tmp;
    __shared__ unsigned long long s_err;  // 2 i (+1: zero duration) of the first failing step, or 2 m + 1 (descent)
    __shared__ unsigned long long s_carry;
    const unsigned long long first_desc = fl->first_desc < n ? fl->first_desc : kNone;
    const bool sorted = fl->nan == 0u && first_desc == kNone;
    const size_t S = two_pose ? 1 : m - 1;
    if (threadIdx.x == 0) {
        s_err = kNone;
        s_carry = 0;
    }
    __syncthreads();
    if (two_pose) {
        if (threadIdx.x == 0) {
            if (zero_duration(knots[0], knots[1])) s_err = 1;
            else if (first_desc != kNone) s_err = 2ull * m + 1;
            ends[0] = n;
        }
    } else if (sorted) {
        // boundaries: running maximum of lower_bound(x, knot i + 1) from the start
        for (size_t base = 0; base < S; base += kPlanThreads) {
            const size_t i = base + threadIdx.x;
            unsigned long long b = 0, flag = kNone;
            if (i < S) {
                const T k0 = knots[i], k1 = knots[i + 1];
                b = lower_bound_walk(x, 0, n, k1);
                if (k0 >= k1) flag = 2ull * i;
            }
            unsigned long long bm;
            BS(tmp).InclusiveScan(b, bm, cub::Max());
            bm = bm < s_carry ? s_carry : bm;
            if (i < S) ends[i] = bm;
            if (flag != kNone) atomicMin(&s_err, flag);
            __syncthreads();
            if (threadIdx.x == kPlanThreads - 1) s_carry = bm;
            __syncthreads();
        }
        // range i is [ends[i-1], ends[i]) (the last one runs to n: the tail uses the last segment)
        for (size_t i = threadIdx.x; i < S; i += kPlanThreads) {
            const unsigned long long lo = i ? ends[i - 1] : 0, hi = i + 1 == S ? n : ends[i];
            if (hi > lo && zero_duration(knots[i], knots[i + 1])) atomicMin(&s_err, 2ull * i + 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) ends[S - 1] = n;
    } else if (threadIdx.x == 0) {
        // the reference's walk, literally
        size_t curr = 0;
        unsigned long long e = kNone;
        for (size_t i = 0; i + 1 < m && e == kNone; ++i) {
            if (knots[i] >= knots[i + 1]) {
                e = 2ull * i;
                break;
            }
            const size_t it = lower_bound_walk(x, curr, n, knots[i + 1]);
            ends[i] = it;
            if (it == curr) continue;
            if (zero_duration(knots[i], knots[i + 1])) e = 2ull * i + 1;
            else if (first_desc >= curr && first_desc < it) e = 2ull * m + 1;
            curr = it;
        }
        if (e == kNone && curr < n) {
            if (zero_duration(knots[m - 2], knots[m - 1])) e = 2ull * (m - 2) + 1;
            else if (first_desc >= curr && first_desc < n) e = 2ull * m + 1;
        }
        ends[S - 1] = n;
        s_err = e;
    }
    __syncthreads();
    const unsigned long long e = s_err;
    if (threadIdx.x == 0) {
        if (e == kNone) put_error(err, vals, OB_POSE_OK, 0, 0, 0, 0);
        else if (e == 2ull * m + 1) put_error(err, vals, OB_POSE_DESCENT, static_cast<long long>(first_desc), 0,
                                             raw(x[first_desc]), raw(x[first_desc - 1]));
        else put_error(err, vals, (e & 1) ? OB_POSE_ZERO_DURATION : OB_POSE_KNOT_ORDER, static_cast<long long>(e >> 1),
                       0, 0, 0);
    }
    if (e != kNone) return;
    for (size_t i = threadIdx.x; i < S; i += kPlanThreads) make_seg(knots, poses, i, segs + i);
}

__device__ __forceinline__ void store_pose(double* o, const double* v) {
    for (int k = 0; k < 16; ++k) o[k] = v[k];
}
__device__ __forceinline__ void store_pose(float* o, const double* v) {
    for (int k = 0; k < 16; ++k) o[k] = __double2float_rn(v[k]);
}

// pose at x of segment s: a * exp((x - t0) * scaled_twist), dt in T, then widened
template <typename T>
__device__ __forceinline__ void seg_pose(const Seg& s, T xv, double* out) {
    const T dt = xv - from_raw<T>(s.t0);
    const double d = static_cast<double>(dt);
    double delta[6], E[16];
    for (int k = 0; k < 6; ++k) delta[k] = mul(d, s.tw[k]);
    posev_exp(delta, E);
    mat4_mul(s.a, E, out);
}

template <typename T, typename P>
__global__ void __launch_bounds__(kQThreads) interp_kernel(const T* __restrict__ x, size_t n,
                                                           const size_t* __restrict__ ends, size_t S,
                                                           const Seg* __restrict__ segs, const long long* err,
                                                           P* __restrict__ out, bool vec) {
    constexpr unsigned kRow = 17;  // padded row: a warp's row writes spread over the banks
    __shared__ P rows[kQThreads * kRow];
    if (*err != 0) return;
    const size_t q0 = static_cast<size_t>(blockIdx.x) * kQThreads;
    const size_t j = q0 + threadIdx.x;
    if (j < n) {
        size_t lo = 0, hi = S - 1;  // the first segment whose range ends after j
        while (lo < hi) {
            const size_t mid = (lo + hi) >> 1;
            if (ends[mid] <= j) lo = mid + 1;
            else hi = mid;
        }
        double v[16];
        seg_pose(segs[lo], x[j], v);
        store_pose(rows + threadIdx.x * kRow, v);
    }
    __syncthreads();
    // the block's rows are one contiguous run of 16-byte vectors in `out`
    constexpr unsigned kPer = 16 / sizeof(P);  // pose values per vector
    const size_t nq = n - q0 < kQThreads ? n - q0 : kQThreads;
    const unsigned nv = static_cast<unsigned>(nq * 16 / kPer);
    if (!vec) {  // `out` is not 16-byte aligned: the same run in single values
        for (unsigned t = threadIdx.x; t < nq * 16; t += kQThreads) out[q0 * 16 + t] = rows[(t / 16) * kRow + t % 16];
        return;
    }
    for (unsigned t = threadIdx.x; t < nv; t += kQThreads) {
        const unsigned e = t * kPer, r = e / 16, c = e % 16;
        const P* src = rows + r * kRow + c;
        if constexpr (sizeof(P) == 8) {
            reinterpret_cast<double2*>(out + q0 * 16)[t] = make_double2(src[0], src[1]);
        } else {
            reinterpret_cast<float4*>(out + q0 * 16)[t] = make_float4(src[0], src[1], src[2], src[3]);
        }
    }
}

// ---- frames ----
struct FrameItem {  // one non-empty slot, device memory
    const unsigned long long* ts;
    const uint32_t* status;
    double* poses;
    unsigned w, first_block, slot, vec;  // vec: poses is 16-byte aligned
};

struct FrameState {
    unsigned long long fail_item;  // first item with a descent, kNone: none
    Seg seg;
};

__device__ __forceinline__ double col_time(const FrameItem& f, unsigned c) {
    return mul(static_cast<double>(f.ts[c]), 1e-9);
}

// one block per item: the first valid column whose timestamp is below the previous valid column's
__global__ void __launch_bounds__(kCheckThreads) frame_check_kernel(const FrameItem* items, FrameState* st,
                                                                    unsigned* desc, double t0, const double* x0,
                                                                    double t1, const double* x1) {
    using BS = cub::BlockScan<int, kCheckThreads>;
    __shared__ typename BS::TempStorage tmp;
    __shared__ int s_prev;
    __shared__ unsigned s_first;
    const FrameItem f = items[blockIdx.x];
    if (blockIdx.x == 0 && threadIdx.x == 0) {  // the shared segment (t0, x0) -> (t1, x1)
        double ai[16], r[16], tw[6];
        inverse4(x0, ai);
        mat4_mul(ai, x1, r);
        poseh_log(r, tw);
        const double inv = 1.0 / (t1 - t0);
        for (int k = 0; k < 16; ++k) st->seg.a[k] = x0[k];
        for (int k = 0; k < 6; ++k) st->seg.tw[k] = mul(inv, tw[k]);
        st->seg.t0 = raw(t0);
    }
    if (threadIdx.x == 0) {
        s_prev = -1;
        s_first = UINT_MAX;
    }
    __syncthreads();
    for (unsigned base = 0; base < f.w; base += kCheckThreads) {
        const unsigned c = base + threadIdx.x;
        const bool valid = c < f.w && (f.status[c] & 1u);
        int last;  // the last valid column before c in this tile
        BS(tmp).ExclusiveScan(valid ? static_cast<int>(c) : -1, last, -1, cub::Max());
        const int prev = last >= 0 ? last : s_prev;
        if (valid && prev >= 0 && col_time(f, c) < col_time(f, static_cast<unsigned>(prev))) atomicMin(&s_first, c);
        __syncthreads();
        if (valid) atomicMax(&s_prev, static_cast<int>(c));
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        desc[blockIdx.x] = s_first;
        if (s_first != UINT_MAX) atomicMin(&st->fail_item, static_cast<unsigned long long>(blockIdx.x));
    }
}

// one thread per column of every item before the first failing one; x1 == NULL: the constant pose x0
__global__ void __launch_bounds__(kWriteThreads) frame_write_kernel(const FrameItem* items, unsigned n_items,
                                                                    const FrameState* st, const unsigned* desc,
                                                                    const double* x0, long long* err, long long* vals) {
    const unsigned bid = blockIdx.x;
    unsigned fi = 0;
    {
        unsigned lo = 0, hi = n_items - 1;  // the last item whose first block is <= bid
        while (lo < hi) {
            const unsigned mid = (lo + hi + 1) >> 1;
            if (items[mid].first_block <= bid) lo = mid;
            else hi = mid - 1;
        }
        fi = lo;
    }
    const unsigned long long fail = st ? st->fail_item : kNone;
    if (bid == 0 && threadIdx.x == 0 && err) {
        if (fail == kNone) {
            put_error(err, vals, OB_POSE_OK, 0, 0, 0, 0);
        } else {
            const FrameItem& f = items[fail];
            const unsigned c = desc[fail];
            int p = static_cast<int>(c) - 1;
            while (p >= 0 && !(f.status[p] & 1u)) --p;
            put_error(err, vals, OB_POSE_DESCENT, c, f.slot, raw(col_time(f, c)), raw(col_time(f, p)));
        }
    }
    if (fi >= fail) return;
    const FrameItem& f = items[fi];
    const unsigned c = (bid - f.first_block) * kWriteThreads + threadIdx.x;
    if (c >= f.w || !(f.status[c] & 1u)) return;
    double v[16];
    if (st) seg_pose(st->seg, col_time(f, c), v);
    else for (int k = 0; k < 16; ++k) v[k] = x0[k];
    double* o = f.poses + static_cast<size_t>(c) * 16;
    if (f.vec) {
        for (int k = 0; k < 8; ++k) reinterpret_cast<double2*>(o)[k] = make_double2(v[2 * k], v[2 * k + 1]);
    } else {
        for (int k = 0; k < 16; ++k) o[k] = v[k];
    }
}

std::string fmt_value(long long bits, int x_dtype) {
    char buf[512];
    if (x_dtype == OB_POSE_X_I64) {
        std::snprintf(buf, sizeof buf, "%lld", bits);
    } else {
        double v;
        std::memcpy(&v, &bits, 8);
        std::snprintf(buf, sizeof buf, "%f", v);  // std::to_string(double)
    }
    return buf;
}

// the reference's message for error words (kind, index, frame) and the two values of a descent
ob_status pose_error_status(const long long* w, int x_dtype) {
    switch (w[0]) {
        case OB_POSE_OK: return OB_OK;
        case OB_POSE_KNOT_ORDER:
            return fail(OB_INVALID_ARGUMENT,
                        "input x_known values are not monotonically increasing or values repeated");
        case OB_POSE_ZERO_DURATION: return fail(OB_INVALID_ARGUMENT, "Cannot interpolate with zero duration between poses");
        default:
            return fail(OB_INVALID_ARGUMENT, "x_interp values must be monotonically increasing: " +
                                                 fmt_value(w[3], x_dtype) + " < " + fmt_value(w[4], x_dtype));
    }
}

}  // namespace

}  // namespace ob

using namespace ob;

namespace {

template <typename T, typename P>
cudaError_t launch_interp(const ob_interp_pose_io* io, const void* x, const void* knots, const void* poses_known,
                          void* out, ScanFlags* fl, size_t* ends, Seg* segs, long long* err, long long* vals,
                          int device, cudaStream_t st) {
    const size_t n = io->n, m = io->m, S = io->two_pose ? 1 : m - 1;
    cudaError_t e = cudaMemsetAsync(fl, 0xff, 8, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(&fl->nan, 0, 8, st);
    if (e != cudaSuccess) return e;
    if (n > 0) {
        const unsigned blocks = static_cast<unsigned>(std::min<size_t>((n + 255) / 256, tunables(device).sm_count * 8ull));
        if constexpr (sizeof(T) == 8 && std::is_same<T, double>::value)
            launch(OB_FAM_POSE, scan_kernel_f64, blocks, 256, 0, st, static_cast<const double*>(x), n, fl);
        else
            launch(OB_FAM_POSE, scan_kernel_i64, blocks, 256, 0, st, static_cast<const long long*>(x), n, fl);
    }
    launch(OB_FAM_POSE, plan_kernel<T, P>, 1, kPlanThreads, 0, st, static_cast<const T*>(x), n,
           static_cast<const T*>(knots), m, static_cast<const P*>(poses_known), io->two_pose, fl, ends, segs, err,
           vals);
    if (n > 0)
        launch(OB_FAM_POSE, interp_kernel<T, P>, static_cast<unsigned>((n + kQThreads - 1) / kQThreads), kQThreads, 0,
               st, static_cast<const T*>(x), n, ends, S, segs, err, static_cast<P*>(out),
               (reinterpret_cast<uintptr_t>(out) & 15u) == 0);
    return cudaGetLastError();
}

}  // namespace

extern "C" ob_status ob_interp_pose(const ob_interp_pose_io* io, ob_stream* s) {
    if (!io) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (io->x_dtype != OB_POSE_X_F64 && io->x_dtype != OB_POSE_X_I64)
        return fail(OB_INVALID_ARGUMENT, "x_dtype must be OB_POSE_X_F64 or OB_POSE_X_I64");
    if (io->pose_dtype != OB_F32 && io->pose_dtype != OB_F64)
        return fail(OB_INVALID_ARGUMENT, "pose_dtype must be OB_F32 or OB_F64");
    if (io->two_pose && io->m != 2) return fail(OB_INVALID_ARGUMENT, "the two-pose form takes m == 2");
    if (!io->two_pose && io->m < 2) return fail(OB_INVALID_ARGUMENT, "Not enough evaluation poses for interpolation");
    if (!io->x_known || !io->poses_known || (io->n && (!io->x_interp || !io->poses)))
        return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (io->n > (static_cast<size_t>(1) << 40) || io->m > (static_cast<size_t>(1) << 31))
        return fail(OB_INVALID_ARGUMENT, "too many poses");
    if (!s) {
        ob_status rs = require_device(0);
        return rs != OB_OK ? rs : fail(OB_INVALID_ARGUMENT, "null pointer");
    }
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    const cudaStream_t st = stream_handle(s);
    const bool dev_err = is_device_ptr(io->error);
    if (io->error && !dev_err) return fail(OB_INVALID_ARGUMENT, "the error words must be device memory");
    const size_t psz = io->pose_dtype == OB_F64 ? 8 : 4;
    if (dev_err && io->n && !is_device_ptr(io->poses))
        return fail(OB_INVALID_ARGUMENT, "a device-side error word needs device outputs");
    const size_t n = io->n, m = io->m, S = io->two_pose ? 1 : m - 1;
    Staging stg(st);
    const void* x = stg.in(io->x_interp, n * 8);
    const void* knots = stg.in(io->x_known, m * 8);
    const void* pk = stg.in(io->poses_known, m * 16 * psz);
    void* out = stg.out(io->poses, n * 16 * psz);
    // work: flags (16 B) | error words (5 x 8 B, padded to 48) | ends (S x 8 B) | segments
    const size_t ends_off = 64, seg_off = (ends_off + S * 8 + 15) & ~static_cast<size_t>(15);
    uint8_t* w = stg.scratch<uint8_t>(seg_off + S * sizeof(Seg));
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage interp_pose");
    ScanFlags* fl = reinterpret_cast<ScanFlags*>(w);
    long long* vals = reinterpret_cast<long long*>(w + 16) + 3;
    long long* err = dev_err ? reinterpret_cast<long long*>(io->error) : reinterpret_cast<long long*>(w + 16);
    size_t* ends = reinterpret_cast<size_t*>(w + ends_off);
    Seg* segs = reinterpret_cast<Seg*>(w + seg_off);
    const bool f64 = io->x_dtype == OB_POSE_X_F64;
    cudaError_t e;
    if (f64 && psz == 8) e = launch_interp<double, double>(io, x, knots, pk, out, fl, ends, segs, err, vals, device, st);
    else if (f64) e = launch_interp<double, float>(io, x, knots, pk, out, fl, ends, segs, err, vals, device, st);
    else if (psz == 8) e = launch_interp<long long, double>(io, x, knots, pk, out, fl, ends, segs, err, vals, device, st);
    else e = launch_interp<long long, float>(io, x, knots, pk, out, fl, ends, segs, err, vals, device, st);
    if (e != cudaSuccess) return fail_cuda(e, "interp_pose launch");
    if (dev_err) {
        e = stg.finish();
        return e == cudaSuccess ? OB_OK : fail_cuda(e, "interp_pose");
    }
    long long words[5];
    e = cudaMemcpyAsync(words, w + 16, sizeof words, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "interp_pose error words");
    if (words[0] != OB_POSE_OK) return pose_error_status(words, io->x_dtype);
    e = stg.finish();
    return e == cudaSuccess ? OB_OK : fail_cuda(e, "interp_pose");
}

extern "C" ob_status ob_frames_interp_pose(const ob_frame_poses_item* frames, size_t n_frames, double t0,
                                           const double* x0, double t1, const double* x1, int64_t* error,
                                           ob_stream* s) {
    if ((n_frames && !frames) || !x0) return fail(OB_INVALID_ARGUMENT, "null pointer");
    size_t first_valid = n_frames;
    for (size_t i = 0; i < n_frames; ++i) {
        const ob_frame_poses_item& f = frames[i];
        if (!f.timestamps) continue;
        if (first_valid == n_frames) first_valid = i;
        if (f.w && (!f.status || !f.poses)) return fail(OB_INVALID_ARGUMENT, "null pointer");
        if (f.w > (1u << 24)) return fail(OB_INVALID_ARGUMENT, "too many columns");
    }
    // interp_pose_range's first check, made on the host: the first valid frame throws, nothing is written
    if (x1 && first_valid < n_frames && std::fabs(t1 - t0) < DBL_EPSILON)
        return fail(OB_INVALID_ARGUMENT, "Cannot interpolate with zero duration between poses");
    if (!s) {
        ob_status rs = require_device(0);
        return rs != OB_OK ? rs : fail(OB_INVALID_ARGUMENT, "null pointer");
    }
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    const cudaStream_t st = stream_handle(s);
    const bool dev_err = is_device_ptr(error);
    if (error && !dev_err) return fail(OB_INVALID_ARGUMENT, "the error words must be device memory");
    Staging stg(st);
    std::vector<FrameItem> items;
    unsigned nb = 0;
    for (size_t i = 0; i < n_frames && !stg.error(); ++i) {
        const ob_frame_poses_item& f = frames[i];
        if (!f.timestamps || f.w == 0) continue;
        FrameItem it{};
        if (x1) it.ts = reinterpret_cast<const unsigned long long*>(stg.in(f.timestamps, f.w));
        it.status = stg.in(f.status, f.w);
        it.poses = stg.inout(f.poses, f.w * 16);  // invalid columns keep their bytes
        it.vec = (reinterpret_cast<uintptr_t>(it.poses) & 15u) == 0;
        it.w = static_cast<unsigned>(f.w);
        it.first_block = nb;
        it.slot = static_cast<unsigned>(i);
        nb += static_cast<unsigned>((f.w + kWriteThreads - 1) / kWriteThreads);
        items.push_back(it);
    }
    const double* dx0 = stg.in(x0, 16);
    const double* dx1 = stg.in(x1, 16);
    // work: error words (5 x 8 B, padded to 48) | FrameState | desc.  The item table goes through the stream's
    // table cache: an unchanged set issues no host copy, so a call can be captured in a CUDA graph after one run
    const size_t st_off = 48, desc_off = st_off + sizeof(FrameState);
    uint8_t* w = stg.scratch<uint8_t>(desc_off + items.size() * 4);
    const void* tab = nullptr;
    cudaError_t e = stg.error();
    if (e == cudaSuccess && !items.empty()) e = stream_table(s, 2, items.data(), items.size() * sizeof(FrameItem), &tab);
    if (e != cudaSuccess) return fail_cuda(e, "stage frames_interp_pose");
    long long* err = dev_err ? reinterpret_cast<long long*>(error) : reinterpret_cast<long long*>(w);
    long long* vals = reinterpret_cast<long long*>(w) + 3;
    FrameState* fs = reinterpret_cast<FrameState*>(w + st_off);
    const FrameItem* ditems = static_cast<const FrameItem*>(tab);
    unsigned* desc = reinterpret_cast<unsigned*>(w + desc_off);
    e = cudaMemsetAsync(err, 0, 24, st);
    if (e == cudaSuccess && !items.empty()) {
        if (x1) e = cudaMemsetAsync(&fs->fail_item, 0xff, 8, st);
        if (e != cudaSuccess) return fail_cuda(e, "stage frames_interp_pose");
        if (x1)
            launch(OB_FAM_POSE, frame_check_kernel, static_cast<unsigned>(items.size()), kCheckThreads, 0, st, ditems,
                   fs, desc, t0, dx0, t1, dx1);
        launch(OB_FAM_POSE, frame_write_kernel, nb, kWriteThreads, 0, st, ditems, static_cast<unsigned>(items.size()),
               x1 ? fs : nullptr, desc, dx0, err, vals);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) return fail_cuda(e, "frames_interp_pose launch");
    // host error words: the call waits once, for the words and the host poses together
    long long words[5] = {0, 0, 0, 0, 0};
    const bool read = !dev_err && x1 && !items.empty();
    if (read) stg.check(cudaMemcpyAsync(words, w, sizeof words, cudaMemcpyDeviceToHost, st));
    e = read ? stg.flush() : stg.finish();
    if (e == cudaSuccess && read) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "frames_interp_pose");
    return pose_error_status(words, OB_POSE_X_F64);
}
