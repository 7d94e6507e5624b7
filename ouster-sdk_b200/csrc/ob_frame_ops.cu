// ob_frame_ops.cu -- frame operations (DESIGN f-10): clip, filter_field, filter_uv, mask and filter_xyz of
// ouster_core/src/frame_ops.cpp / python/src/ouster/sdk/core/frame_ops.py as one masked write over the pixel
// fields of a batch of frames, and select_by_index / reduce_by_factor as one row gather.
//
// Masked write.  A thread owns a run of kRun consecutive pixels of one frame (flat row-major index, so a run
// may wrap onto the next row; the predicate derives (row, col) per pixel).  It evaluates the predicate once per
// return, then walks the frame's field table: a target whose run has no hit is not touched at all, the others are
// loaded (16-byte vectors when the run is aligned and whole), merged with the target's fill pattern and stored
// back chunk by chunk, only where a byte changes.  One thread owns a pixel across every field, so a source that
// is also a target is read before any write to it.  The fill pattern is static_cast<T>(invalid), computed on the
// host per field, so the write itself is type-agnostic; only clip and a filter_field source read values as T.
//
// Row gather.  One launch copies the selected rows of every pixel field of every frame, in the widest unit that
// the source, destination and row length are all aligned to.
//
// Both launches take their tables (fields, frame ranges, reduced shifts, selected rows) as kernel parameters, so
// nothing is uploaded or synchronised per call and a call on device frames can be captured in a CUDA graph.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "ob_api_common.h"
#include "ob_project.cuh"

namespace ob {
namespace {

constexpr int kRun = 16;            // pixels per thread
constexpr int kThreads = 256;
constexpr int kMaxShiftRows = 2048; // rows a destaggered-column predicate can take (shifts travel as parameters)

struct MaskEntry {
    void* data;
    uint64_t fill;      // bit pattern of static_cast<T>(invalid) (0 for OB_FRAME_ZERO)
    uint8_t type;       // ChanFieldType tag
    uint8_t role;       // ob_frame_role
    uint16_t esize;     // bytes per element: 1, 2, 4 or 8 (OB_FRAME_ZERO: any size of one pixel)
    uint32_t frame;
};

template <int CAP>
struct MaskParams {
    uint32_t h, w, npx, n_entries;
    int32_t pred, axis, lut_f64, has_poses;
    double lo, hi;
    const void* dir;
    const void* off;
    const void* poses;     // n_frames x w x 16 of the LUT dtype, or null
    uint32_t frame0;       // frame index of blockIdx.y == 0
    uint16_t begin[CAP + 1];  // entries of frame (frame0 + y) are [begin[y], begin[y + 1])
    MaskEntry e[CAP];
    uint16_t shift[kMaxShiftRows];  // COLS: shift[r] mod w
};

// axis coordinate of lut(range) at pixel i of frame f, posed by column c when poses are given; compared in T
template <typename T, int CAP>
__device__ __forceinline__ bool xyz_range_hit(const MaskParams<CAP>& p, const uint32_t* rng, uint32_t f, size_t i,
                                              uint32_t c) {
    const T* d = static_cast<const T*>(p.dir) + i * 3;
    const T* o = static_cast<const T*>(p.off) + i * 3;
    const uint32_t r = __ldg(rng + i);
    T v;
    if (p.has_poses) {
        const T x = project(r, __ldg(d), __ldg(o)), y = project(r, __ldg(d + 1), __ldg(o + 1)),
                z = project(r, __ldg(d + 2), __ldg(o + 2));
        const T* m = static_cast<const T*>(p.poses) + (size_t(f) * p.w + c) * 16 + 4 * p.axis;
        T mm[4] = {__ldg(m), __ldg(m + 1), __ldg(m + 2), __ldg(m + 3)};
        v = pose_row(mm, x, y, z);
    } else {
        v = project(r, __ldg(d + p.axis), __ldg(o + p.axis));
    }
    return v >= static_cast<T>(p.lo) && v <= static_cast<T>(p.hi);
}

template <typename T>
__device__ __forceinline__ bool xyz_points_hit(const void* pts, size_t i, int axis, double lo, double hi) {
    const T v = static_cast<const T*>(pts)[i * 3 + axis];
    return v >= static_cast<T>(lo) && v <= static_cast<T>(hi);
}

// hit bits (bit k: pixel idx0 + k) of one return's predicate
template <int CAP>
__device__ uint32_t predicate_bits(const MaskParams<CAP>& p, const MaskEntry* src, uint32_t f, size_t idx0, int n) {
    uint32_t bits = 0;
    uint32_t r = uint32_t(idx0 / p.w), c = uint32_t(idx0 - size_t(r) * p.w);
    for (int k = 0; k < n; ++k) {
        const size_t i = idx0 + k;
        bool hit = false;
        switch (p.pred) {
            case OB_FRAME_ROWS: hit = double(r) >= p.lo && double(r) < p.hi; break;
            case OB_FRAME_COLS: {
                uint32_t cc = c + p.shift[r];
                if (cc >= p.w) cc -= p.w;
                hit = double(cc) >= p.lo && double(cc) < p.hi;
                break;
            }
            case OB_FRAME_XYZ_RANGE:
                hit = p.lut_f64 ? xyz_range_hit<double>(p, static_cast<const uint32_t*>(src->data), f, i, c)
                                : xyz_range_hit<float>(p, static_cast<const uint32_t*>(src->data), f, i, c);
                break;
            case OB_FRAME_XYZ_POINTS:
                hit = src->type == 10 ? xyz_points_hit<double>(src->data, i, p.axis, p.lo, p.hi)
                                      : xyz_points_hit<float>(src->data, i, p.axis, p.lo, p.hi);
                break;
            default: break;
        }
        bits |= uint32_t(hit) << k;
        if (++c == p.w) {
            c = 0;
            ++r;
        }
    }
    return bits;
}

// bit k set where lo <= (double)v <= hi for pixel idx0 + k (NaN: clear); whole aligned runs load 16-byte chunks.
// Plain loads: a clip target or a filter_field source may be written later in this launch, by this thread only.
template <typename T>
__device__ __forceinline__ uint32_t in_range_bits_t(const void* data, size_t idx0, int n, double lo, double hi) {
    const T* base = static_cast<const T*>(data) + idx0;
    uint32_t bits = 0;
    if (n == kRun && (reinterpret_cast<uintptr_t>(base) & 15) == 0) {
        constexpr int kPer = 16 / sizeof(T);
        const uint4* vb = reinterpret_cast<const uint4*>(base);
#pragma unroll
        for (int ch = 0; ch < kRun / kPer; ++ch) {
            const uint4 v = vb[ch];
            const T* u = reinterpret_cast<const T*>(&v);
#pragma unroll
            for (int k = 0; k < kPer; ++k) {
                const double d = static_cast<double>(u[k]);
                bits |= uint32_t(d >= lo && d <= hi) << (ch * kPer + k);
            }
        }
        return bits;
    }
    for (int k = 0; k < n; ++k) {
        const double d = static_cast<double>(base[k]);
        bits |= uint32_t(d >= lo && d <= hi) << k;
    }
    return bits;
}

__device__ uint32_t in_range_bits(const void* data, int type, size_t idx0, int n, double lo, double hi) {
    switch (type) {
        case 1: return in_range_bits_t<uint8_t>(data, idx0, n, lo, hi);
        case 2: return in_range_bits_t<uint16_t>(data, idx0, n, lo, hi);
        case 3: return in_range_bits_t<uint32_t>(data, idx0, n, lo, hi);
        case 4: return in_range_bits_t<unsigned long long>(data, idx0, n, lo, hi);   // cvt.rn.f64.u64
        case 5: return in_range_bits_t<int8_t>(data, idx0, n, lo, hi);
        case 6: return in_range_bits_t<int16_t>(data, idx0, n, lo, hi);
        case 7: return in_range_bits_t<int32_t>(data, idx0, n, lo, hi);
        case 8: return in_range_bits_t<long long>(data, idx0, n, lo, hi);            // cvt.rn.f64.s64
        case 9: return in_range_bits_t<float>(data, idx0, n, lo, hi);
        default: return in_range_bits_t<double>(data, idx0, n, lo, hi);
    }
}

// write fill where bit k is set; whole aligned runs move in 16-byte chunks and store only chunks that change
template <typename U>
__device__ __forceinline__ void masked_write(void* data, size_t idx0, int n, uint32_t bits, uint64_t fill64) {
    U* base = static_cast<U*>(data) + idx0;
    const U fill = static_cast<U>(fill64);
    if (n == kRun && (reinterpret_cast<uintptr_t>(base) & 15) == 0) {
        constexpr int kPer = 16 / sizeof(U);  // elements per chunk
        uint4* vb = reinterpret_cast<uint4*>(base);
#pragma unroll
        for (int ch = 0; ch < kRun / kPer; ++ch) {
            const uint32_t cb = (bits >> (ch * kPer)) & ((1u << kPer) - 1u);
            if (!cb) continue;
            uint4 v = vb[ch];
            U* u = reinterpret_cast<U*>(&v);
            bool changed = false;
#pragma unroll
            for (int k = 0; k < kPer; ++k) {
                if ((cb >> k) & 1u) {
                    changed |= u[k] != fill;
                    u[k] = fill;
                }
            }
            if (changed) vb[ch] = v;
        }
        return;
    }
    for (int k = 0; k < n; ++k)
        if (((bits >> k) & 1u) && base[k] != fill) base[k] = fill;
}

__device__ __forceinline__ void write_entry(const MaskEntry& e, size_t idx0, int n, uint32_t bits) {
    if (!bits) return;
    switch (e.esize) {
        case 1: masked_write<uint8_t>(e.data, idx0, n, bits, e.fill); break;
        case 2: masked_write<uint16_t>(e.data, idx0, n, bits, e.fill); break;
        case 4: masked_write<uint32_t>(e.data, idx0, n, bits, e.fill); break;
        case 8: masked_write<unsigned long long>(e.data, idx0, n, bits, e.fill); break;
        default: {  // zero-fill of pixels of another size (a skipped type with extra dims): bytewise
            uint8_t* b = static_cast<uint8_t*>(e.data) + idx0 * e.esize;
            for (size_t k = 0, nb = size_t(n) * e.esize; k < nb; ++k)
                if (b[k]) b[k] = 0;
            break;
        }
    }
}

template <int CAP>
__global__ void __launch_bounds__(kThreads) frame_mask_kernel(const __grid_constant__ MaskParams<CAP> p) {
    const size_t idx0 = (size_t(blockIdx.x) * kThreads + threadIdx.x) * kRun;
    if (idx0 >= p.npx) return;
    const int n = p.npx - idx0 < size_t(kRun) ? int(p.npx - idx0) : kRun;
    const uint32_t y = blockIdx.y, f = p.frame0 + y;
    const int b = p.begin[y], end = p.begin[y + 1];
    uint32_t bits[2] = {0u, 0u};
    if (p.pred != OB_FRAME_CLIP) {
        const MaskEntry* src[2] = {nullptr, nullptr};
        for (int j = b; j < end; ++j) {
            if (p.e[j].role == OB_FRAME_SOURCE) src[0] = &p.e[j];
            if (p.e[j].role == OB_FRAME_SOURCE2) src[1] = &p.e[j];
        }
        if (p.pred == OB_FRAME_VALUE) {
            for (int r = 0; r < 2; ++r)
                if (src[r]) bits[r] = in_range_bits(src[r]->data, src[r]->type, idx0, n, p.lo, p.hi);
        } else if (p.pred == OB_FRAME_ROWS || p.pred == OB_FRAME_COLS) {
            bits[0] = bits[1] = predicate_bits(p, nullptr, f, idx0, n);
        } else {
            for (int r = 0; r < 2; ++r)
                if (src[r]) bits[r] = predicate_bits(p, src[r], f, idx0, n);
        }
    }
    const uint32_t all = (1u << n) - 1u;   // clip: hit where the value is outside [lo, hi] or NaN
    for (int j = b; j < end; ++j) {
        const MaskEntry& e = p.e[j];
        switch (e.role) {
            case OB_FRAME_TARGET:
                write_entry(e, idx0, n, p.pred == OB_FRAME_CLIP ? ~in_range_bits(e.data, e.type, idx0, n, p.lo, p.hi) & all
                                                        : bits[0]);
                break;
            case OB_FRAME_TARGET2: write_entry(e, idx0, n, bits[1]); break;
            case OB_FRAME_ZERO: write_entry(e, idx0, n, all); break;   // a field type the per-type visit skips
            default: break;
        }
    }
}

// ---- row gather ----
struct RowEntry {
    const void* src;
    void* dst;
    uint32_t row_bytes;
    uint32_t unit;   // 16, 8, 4, 2 or 1
};

template <int CAP>
struct RowParams {
    uint32_t n_entries, n_rows;
    RowEntry e[CAP];
    uint32_t rows[kMaxShiftRows];
};

template <typename V, int CAP>
__device__ __forceinline__ void gather_rows(const RowParams<CAP>& p, const RowEntry& e) {
    const uint32_t per_row = e.row_bytes / sizeof(V);
    const size_t total = size_t(per_row) * p.n_rows;
    const V* s = static_cast<const V*>(e.src);
    V* d = static_cast<V*>(e.dst);
    for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < total; u += size_t(gridDim.x) * blockDim.x) {
        const uint32_t row = uint32_t(u / per_row), k = uint32_t(u - size_t(row) * per_row);
        d[u] = s[size_t(p.rows[row]) * per_row + k];
    }
}

template <int CAP>
__global__ void __launch_bounds__(kThreads) frame_rows_kernel(const __grid_constant__ RowParams<CAP> p) {
    const RowEntry& e = p.e[blockIdx.y];
    switch (e.unit) {
        case 16: gather_rows<uint4>(p, e); break;
        case 8: gather_rows<uint2>(p, e); break;
        case 4: gather_rows<uint32_t>(p, e); break;
        case 2: gather_rows<uint16_t>(p, e); break;
        default: gather_rows<uint8_t>(p, e); break;
    }
}

// ---- host side ----
size_t type_size(int t) {
    switch (t) {
        case 1: case 5: return 1;
        case 2: case 6: case 12: return 2;
        case 3: case 7: case 9: return 4;
        case 4: case 8: case 10: return 8;
        default: return 0;
    }
}
bool handled(int t) { return t >= 1 && t <= 10; }

// static_cast<T>(invalid) as T's bit pattern; false where the reference's cast is undefined
bool fill_pattern(int type, double v, uint64_t* out) {
    auto int_fill = [&](double lo, double hi, auto tag) {
        using I = decltype(tag);
        if (!std::isfinite(v)) return false;
        const double t = std::trunc(v);
        if (!(t >= lo && t <= hi)) return false;
        I x = static_cast<I>(t);
        uint64_t bits = 0;
        std::memcpy(&bits, &x, sizeof(I));
        *out = bits;
        return true;
    };
    switch (type) {
        case 1: return int_fill(0.0, 255.0, uint8_t{});
        case 2: return int_fill(0.0, 65535.0, uint16_t{});
        case 3: return int_fill(0.0, 4294967295.0, uint32_t{});
        case 4: return int_fill(0.0, 18446744073709549568.0, uint64_t{});   // largest double below 2^64
        case 5: return int_fill(-128.0, 127.0, int8_t{});
        case 6: return int_fill(-32768.0, 32767.0, int16_t{});
        case 7: return int_fill(-2147483648.0, 2147483647.0, int32_t{});
        case 8: return int_fill(-9223372036854775808.0, 9223372036854774784.0, int64_t{});
        case 9: {
            const float x = static_cast<float>(v);
            uint32_t b;
            std::memcpy(&b, &x, 4);
            *out = b;
            return true;
        }
        case 10: std::memcpy(out, &v, 8); return true;
        default: return false;
    }
}

template <int CAP>
cudaError_t launch_mask(MaskParams<CAP>& p, const std::vector<MaskEntry>& ents, const std::vector<uint32_t>& fbeg,
                        uint32_t f0, uint32_t f1, cudaStream_t st) {
    p.frame0 = f0;
    const uint32_t e0 = fbeg[f0];
    p.n_entries = fbeg[f1] - e0;
    for (uint32_t f = f0; f <= f1; ++f) p.begin[f - f0] = uint16_t(fbeg[f] - e0);
    std::copy(ents.begin() + e0, ents.begin() + fbeg[f1], p.e);
    const size_t runs = (size_t(p.npx) + kRun - 1) / kRun;
    dim3 grid(unsigned((runs + kThreads - 1) / kThreads), f1 - f0);
    launch(OB_FAM_FRAME_OPS, frame_mask_kernel<CAP>, grid, kThreads, 0, st, p);
    return cudaGetLastError();
}

template <int CAP>
cudaError_t launch_rows(RowParams<CAP>& p, const RowEntry* ents, uint32_t n, cudaStream_t st, uint32_t max_units) {
    p.n_entries = n;
    std::copy(ents, ents + n, p.e);
    const unsigned gx = unsigned(std::min<size_t>((size_t(max_units) + kThreads - 1) / kThreads, 4096));
    launch(OB_FAM_FRAME_OPS, frame_rows_kernel<CAP>, dim3(std::max(gx, 1u), n), kThreads, 0, st, p);
    return cudaGetLastError();
}

}  // namespace
}  // namespace ob

using namespace ob;

extern "C" {

ob_status ob_frame_mask_fields(const ob_frame_ops_io* io, ob_stream* s) {
    if (!io || !s || (io->n_fields && !io->fields)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const ob_frame_ops_io& a = *io;
    if (a.predicate < OB_FRAME_CLIP || a.predicate > OB_FRAME_XYZ_POINTS)
        return fail(OB_INVALID_ARGUMENT, "unknown frame predicate");
    if (a.n_frames > 65535) return fail(OB_INVALID_ARGUMENT, "too many frames for one call");
    const size_t npx = size_t(a.h) * a.w;
    if (npx > 0xffffffffull) return fail(OB_INVALID_ARGUMENT, "frame too large");
    if ((a.predicate == OB_FRAME_XYZ_RANGE || a.predicate == OB_FRAME_XYZ_POINTS) && (a.axis < 0 || a.axis > 2))
        return fail(OB_INVALID_ARGUMENT, "axis_idx must be in the range [0, 2]");
    if (a.predicate == OB_FRAME_COLS && (a.h > kMaxShiftRows || (a.h && !a.pixel_shift_by_row)))
        return fail(OB_INVALID_ARGUMENT, "pixel_shift_by_row must have one entry per row (at most 2048 rows)");
    // validate every entry before anything is launched: a failing call modifies nothing
    std::vector<std::vector<MaskEntry>> per_frame(a.n_frames);
    for (size_t i = 0; i < a.n_fields; ++i) {
        const ob_frame_field& fd = a.fields[i];
        if (fd.frame >= a.n_frames) return fail(OB_INVALID_ARGUMENT, "field entry names a frame outside the batch");
        if (!fd.data && npx) return fail(OB_INVALID_ARGUMENT, "null pointer");
        MaskEntry e{};
        e.data = fd.data;
        e.type = uint8_t(fd.type);
        e.role = uint8_t(fd.role);
        e.frame = fd.frame;
        switch (fd.role) {
            case OB_FRAME_TARGET:
            case OB_FRAME_TARGET2:
                if (!handled(fd.type)) return fail(OB_INVALID_ARGUMENT, "target field type is not a numeric pixel type");
                if (!fill_pattern(fd.type, a.invalid, &e.fill))
                    return fail(OB_INVALID_ARGUMENT, "invalid value cannot be represented in the field's type");
                e.esize = uint16_t(type_size(fd.type));
                break;
            case OB_FRAME_ZERO: {
                const size_t es = fd.elem_bytes;
                if (es == 0 || es > 65535)
                    return fail(OB_INVALID_ARGUMENT, "zero-filled field needs 1 to 65535 bytes per pixel");
                e.esize = uint16_t(es);
                e.fill = 0;
                break;
            }
            case OB_FRAME_SOURCE:
            case OB_FRAME_SOURCE2:
                if (a.predicate == OB_FRAME_VALUE && !handled(fd.type))
                    return fail(OB_INVALID_ARGUMENT, "filter_field requires a pixel field with shape (h, w) to build a mask");
                if (a.predicate == OB_FRAME_XYZ_RANGE && fd.type != 3)
                    return fail(OB_INVALID_ARGUMENT, "range must be uint32");
                if (a.predicate == OB_FRAME_XYZ_POINTS && fd.type != 9 && fd.type != 10)
                    return fail(OB_INVALID_ARGUMENT, "points must be float32 or float64");
                break;
            default: return fail(OB_INVALID_ARGUMENT, "unknown field role");
        }
        per_frame[fd.frame].push_back(e);
        if (per_frame[fd.frame].size() > 512) return fail(OB_INVALID_ARGUMENT, "too many fields in one frame");
    }
    LutView lut{};
    if (a.predicate == OB_FRAME_XYZ_RANGE) {
        if (!a.lut) return fail(OB_INVALID_ARGUMENT, "null pointer");
        lut = lut_view(a.lut);
        if (lut.h != a.h || lut.w != a.w) return fail(OB_INVALID_ARGUMENT, "Frame dimensions do not match lut.");
        if (lut.device != stream_device(s)) return fail(OB_INVALID_ARGUMENT, "stream and lut are on different devices");
    }
    ob_status rs = require_device(stream_device(s));
    if (rs != OB_OK) return rs;
    if (npx == 0 || a.n_frames == 0 || a.n_fields == 0) return OB_OK;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    bool host_io = false;
    // stage host buffers: targets in and out, sources in
    std::vector<MaskEntry> ents;
    std::vector<uint32_t> fbeg(a.n_frames + 1, 0);
    for (uint32_t f = 0; f < a.n_frames && !stg.error(); ++f) {
        fbeg[f] = uint32_t(ents.size());
        for (MaskEntry m : per_frame[f]) {
            const bool src = m.role == OB_FRAME_SOURCE || m.role == OB_FRAME_SOURCE2;
            const size_t bytes = npx * (src ? (a.predicate == OB_FRAME_XYZ_POINTS ? 3 * type_size(m.type)
                                                                              : type_size(m.type))
                                            : m.esize);
            if (!is_device_ptr(m.data)) {
                host_io |= !src;
                m.data = src ? const_cast<void*>(stg.in(m.data, bytes)) : stg.inout(m.data, bytes);
            }
            ents.push_back(m);
        }
    }
    fbeg[a.n_frames] = uint32_t(ents.size());
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage frame fields");
    const void* dposes = nullptr;
    if (a.predicate == OB_FRAME_XYZ_RANGE && a.poses) {
        dposes = stg.in(a.poses, size_t(a.n_frames) * a.w * 16 * (lut.dtype == OB_F64 ? 8 : 4));
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage poses");
    }
    std::vector<uint16_t> sh;
    if (a.predicate == OB_FRAME_COLS) reduce_shifts(a.pixel_shift_by_row, a.h, a.w, 0, sh);

    // frames go to one launch while their entries fit the parameter table; a second table size keeps the
    // parameter block of a single-frame call small
    auto fill = [&](auto& p) {
        p.h = a.h;
        p.w = a.w;
        p.npx = uint32_t(npx);
        p.pred = a.predicate;
        p.axis = a.axis;
        p.lut_f64 = lut.dtype == OB_F64;
        p.has_poses = dposes != nullptr;
        p.lo = a.lower;
        p.hi = a.upper;
        p.dir = lut.dir;
        p.off = lut.off;
        p.poses = dposes;
        for (size_t r = 0; r < sh.size(); ++r) p.shift[r] = sh[r];
    };
    constexpr int kSmall = 32, kLarge = 512;
    cudaError_t e = cudaSuccess;
    if (ents.size() <= size_t(kSmall) && a.n_frames <= uint32_t(kSmall)) {
        auto p = std::make_unique<MaskParams<kSmall>>();
        fill(*p);
        e = launch_mask(*p, ents, fbeg, 0, a.n_frames, st);
    } else {
        auto p = std::make_unique<MaskParams<kLarge>>();
        fill(*p);
        uint32_t f0 = 0;
        while (f0 < a.n_frames && e == cudaSuccess) {
            uint32_t f1 = f0 + 1;
            while (f1 < a.n_frames && f1 - f0 < uint32_t(kLarge) && fbeg[f1 + 1] - fbeg[f0] <= uint32_t(kLarge)) ++f1;
            e = launch_mask(*p, ents, fbeg, f0, f1, st);
            f0 = f1;
        }
    }
    stg.check(e);
    e = stg.flush();
    if (e == cudaSuccess && host_io) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "frame mask");
    return OB_OK;
}

ob_status ob_frame_select_rows(const ob_frame_rows_io* io, ob_stream* s) {
    if (!io || !s || (io->n_entries && !io->entries) || (io->n_rows && !io->rows))
        return fail(OB_INVALID_ARGUMENT, "null pointer");
    const ob_frame_rows_io& a = *io;
    if (a.n_rows > kMaxShiftRows) return fail(OB_INVALID_ARGUMENT, "too many rows for one call");
    for (uint32_t i = 0; i < a.n_entries; ++i) {
        const ob_frame_rows_entry& r = a.entries[i];
        if ((!r.src || !r.dst) && r.row_bytes) return fail(OB_INVALID_ARGUMENT, "null pointer");
        if (r.row_bytes > 0xffffffffull) return fail(OB_INVALID_ARGUMENT, "row too large");
        for (uint32_t k = 0; k < a.n_rows; ++k)
            if (a.rows[k] >= r.src_rows) return fail(OB_INVALID_ARGUMENT, "row index out of range");
    }
    ob_status rs = require_device(stream_device(s));
    if (rs != OB_OK) return rs;
    if (a.n_entries == 0 || a.n_rows == 0) return OB_OK;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    bool host_io = false;
    std::vector<RowEntry> ents;
    uint32_t max_units = 0;
    for (uint32_t i = 0; i < a.n_entries && !stg.error(); ++i) {
        const ob_frame_rows_entry& r = a.entries[i];
        if (!r.row_bytes) continue;
        RowEntry x{r.src, r.dst, uint32_t(r.row_bytes), 1};
        if (!is_device_ptr(r.src)) x.src = stg.in(r.src, r.src_rows * r.row_bytes);
        if (!stg.error() && !is_device_ptr(r.dst)) {
            host_io = true;
            x.dst = stg.out(r.dst, size_t(a.n_rows) * r.row_bytes);
        }
        const uintptr_t al = reinterpret_cast<uintptr_t>(x.src) | reinterpret_cast<uintptr_t>(x.dst) | x.row_bytes;
        x.unit = (al & 15) == 0 ? 16 : (al & 7) == 0 ? 8 : (al & 3) == 0 ? 4 : (al & 1) == 0 ? 2 : 1;
        max_units = std::max(max_units, uint32_t(std::min<size_t>(size_t(x.row_bytes / x.unit) * a.n_rows, 0xffffffffu)));
        ents.push_back(x);
    }
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage frame rows");
    constexpr int kCap = 768;   // 18 KB of entries + 8 KB of rows: within the 32 KB parameter limit
    auto p = std::make_unique<RowParams<kCap>>();
    p->n_rows = a.n_rows;
    for (uint32_t k = 0; k < a.n_rows; ++k) p->rows[k] = a.rows[k];
    cudaError_t e = cudaSuccess;
    for (size_t b = 0; b < ents.size() && e == cudaSuccess; b += kCap) {
        const uint32_t n = uint32_t(std::min<size_t>(kCap, ents.size() - b));
        e = launch_rows(*p, ents.data() + b, n, st, max_units);
    }
    stg.check(e);
    e = stg.flush();
    if (e == cudaSuccess && host_io) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "frame select rows");
    return OB_OK;
}

}  // extern "C"
