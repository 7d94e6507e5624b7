// ob_map_rows.cu -- frame -> map rows (DESIGN f-11): the map exporter's per-return step in ONE launch.
//
// What it replaces (reference paths relative to the reference tree):
//   python/src/ouster/cli/plugins/map_export.py:589-617, per return of a frame:
//     valid = range > 0; dewarp(xyzlut_double(range), body_to_world)[valid] and every requested field [valid],
//     np.concatenate(..., axis=1).astype(float64), then VoxelHashMapXd.add_points
//
// A CTA owns 1024 consecutive pixels (row-major, staggered) of one item; a thread owns 4 of them.  The CTA counts
// its pixels with range > 0, scans the counts (cub::BlockScan), takes its base from the decoupled look-back over
// the CTAs before it (ob_lookback.cuh, shared with K3; items simply continue the chain) and writes each surviving
// pixel's row at base + rank: x, y, z from K1's projection and pose code (ob_project.cuh), then the fields'
// channels widened to double.  Widening each value on its own equals the exporter's concatenate-then-astype:
// numpy's common type of the fields holds every one of their values exactly, or is float64 itself.
#include <cuda_fp16.h>

#include <cub/block/block_scan.cuh>

#include <algorithm>
#include <vector>

#include "ob_api_common.h"
#include "ob_lookback.cuh"
#include "ob_project.cuh"

namespace ob {
namespace {

constexpr unsigned kMaxMapFields = 16;
constexpr unsigned kMrThreads = 256, kMrPix = 4, kMrTile = kMrThreads * kMrPix;

struct MrField {
    const void* data;  // h x w x channels
    int32_t type;      // ChanFieldType tag
    uint32_t channels;
};

struct MrItem {  // one per item of the launch, device memory
    const uint32_t* range;
    const double* dir;
    const double* off;
    const double* poses;  // W x 16
    unsigned long long n_px;
    unsigned W, first_block, n_blocks, n_fields;
    MrField f[kMaxMapFields];
};

// bytes of one value of a ChanFieldType tag, 0 for tags a map row cannot hold
size_t field_bytes(int32_t type) {
    switch (type) {
        case 1: case 5: return 1;
        case 2: case 6: case 12: return 2;
        case 3: case 7: case 9: return 4;
        case 4: case 8: case 10: return 8;
        default: return 0;
    }
}

__device__ __forceinline__ double widen(const void* p, int32_t type, size_t i) {
    switch (type) {
        case 1: return static_cast<double>(static_cast<const uint8_t*>(p)[i]);
        case 2: return static_cast<double>(static_cast<const uint16_t*>(p)[i]);
        case 3: return static_cast<double>(static_cast<const uint32_t*>(p)[i]);
        case 4: return static_cast<double>(static_cast<const unsigned long long*>(p)[i]);
        case 5: return static_cast<double>(static_cast<const int8_t*>(p)[i]);
        case 6: return static_cast<double>(static_cast<const int16_t*>(p)[i]);
        case 7: return static_cast<double>(static_cast<const int32_t*>(p)[i]);
        case 8: return static_cast<double>(static_cast<const long long*>(p)[i]);
        case 9: return static_cast<double>(static_cast<const float*>(p)[i]);
        case 10: return static_cast<const double*>(p)[i];
        default: return static_cast<double>(__half2float(__ushort_as_half(static_cast<const uint16_t*>(p)[i])));
    }
}

__global__ void __launch_bounds__(kMrThreads) map_rows_kernel(const MrItem* __restrict__ items, unsigned n_items,
                                                              unsigned cols, unsigned* ticket, Lookback lb,
                                                              unsigned long long* item_end, double* __restrict__ out,
                                                              unsigned long long capacity) {
    using BS = cub::BlockScan<unsigned, kMrThreads>;
    __shared__ typename BS::TempStorage tmp;
    __shared__ unsigned s_bid;
    __shared__ unsigned long long s_excl;
    if (threadIdx.x == 0) s_bid = atomicAdd(ticket, 1u);
    __syncthreads();
    const unsigned bid = s_bid;
    unsigned f = 0;
    while (f + 1 < n_items && items[f + 1].first_block <= bid) ++f;
    const MrItem& it = items[f];
    const unsigned long long p0 =
        static_cast<unsigned long long>(bid - it.first_block) * kMrTile + threadIdx.x * kMrPix;
    uint32_t r[kMrPix];
    unsigned c = 0;
#pragma unroll
    for (unsigned j = 0; j < kMrPix; ++j) {
        r[j] = p0 + j < it.n_px ? it.range[p0 + j] : 0u;
        c += r[j] != 0u ? 1u : 0u;
    }
    unsigned rank, total;
    BS(tmp).ExclusiveSum(c, rank, total);
    if (threadIdx.x < 32) {
        const unsigned long long excl = lookback_exclusive(lb, bid, total, threadIdx.x);
        if (threadIdx.x == 0) {
            s_excl = excl;
            if (bid + 1 == it.first_block + it.n_blocks) item_end[f] = excl + total;
        }
    }
    __syncthreads();
    unsigned long long w = s_excl + rank;
    for (unsigned j = 0; j < kMrPix; ++j) {
        if (r[j] == 0u) continue;
        if (w < capacity) {
            const unsigned long long px = p0 + j;
            const double* m = it.poses + static_cast<size_t>(px % it.W) * 16;
            const double x = project(r[j], it.dir[px * 3], it.off[px * 3]);
            const double y = project(r[j], it.dir[px * 3 + 1], it.off[px * 3 + 1]);
            const double z = project(r[j], it.dir[px * 3 + 2], it.off[px * 3 + 2]);
            double* o = out + w * cols;
            o[0] = pose_row(m, x, y, z);
            o[1] = pose_row(m + 4, x, y, z);
            o[2] = pose_row(m + 8, x, y, z);
            unsigned k = 3;
            for (unsigned fi = 0; fi < it.n_fields; ++fi) {
                const MrField& fd = it.f[fi];
                for (unsigned ch = 0; ch < fd.channels; ++ch) o[k++] = widen(fd.data, fd.type, px * fd.channels + ch);
            }
        }
        ++w;
    }
}

// scratch: [ticket + pad : 16 B][state u32 x nb, padded to 8][agg u64 x nb][incl u64 x nb][item_end u64 x ni]
size_t state_bytes(unsigned nb) { return 16 + ((static_cast<size_t>(nb) * 4 + 7) & ~static_cast<size_t>(7)); }

}  // namespace
}  // namespace ob

using namespace ob;

extern "C" ob_status ob_frames_to_map_rows(const ob_map_rows_item* items, size_t n_items, double* rows, size_t cols,
                                           size_t capacity, size_t* n_rows, ob_stream* s) {
    if (!s || !n_rows || (n_items && !items)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    const cudaStream_t st = stream_handle(s);
    Staging stg(st);
    CountedRows res(n_rows, capacity, stg, st, "map rows count");
    rs = res.zero();
    if (rs == OB_OK) rs = res.refuse({rows}, "a device-side count needs device outputs");
    if (rs != OB_OK) return rs;
    // every check before anything is staged
    for (size_t i = 0; i < n_items; ++i) {
        const ob_map_rows_item& io = items[i];
        if (!io.lut || !io.range || !io.poses || (io.n_fields && !io.fields))
            return fail(OB_INVALID_ARGUMENT, "null lut / range / poses / fields");
        const LutView lv = lut_view(io.lut);
        if (lv.dtype != OB_F64) return fail(OB_INVALID_ARGUMENT, "map rows need a float64 lut");
        if (lv.device != device) return fail(OB_INVALID_ARGUMENT, "lut and stream are on different devices");
        if (io.n_fields > kMaxMapFields) return fail(OB_INVALID_ARGUMENT, "too many fields");
        size_t c = 3;
        for (size_t k = 0; k < io.n_fields; ++k) {
            const ob_map_field& fd = io.fields[k];
            if (field_bytes(fd.type) == 0) return fail(OB_INVALID_ARGUMENT, "unknown field type");
            if (fd.channels < 1) return fail(OB_INVALID_ARGUMENT, "field channels must be at least 1");
            if (!fd.data) return fail(OB_INVALID_ARGUMENT, "null lut / range / poses / fields");
            c += fd.channels;
        }
        if (c != cols) return fail(OB_INVALID_ARGUMENT, "cols must be 3 plus the channels of every item's fields");
    }
    if (capacity && !rows) return fail(OB_INVALID_ARGUMENT, "null rows buffer");
    std::vector<MrItem> hi;
    unsigned nb = 0;
    for (size_t i = 0; i < n_items; ++i) {
        const ob_map_rows_item& io = items[i];
        const LutView lv = lut_view(io.lut);
        const size_t n_px = lv.h * lv.w;
        if (n_px == 0) continue;
        MrItem it{};
        it.dir = static_cast<const double*>(lv.dir);
        it.off = static_cast<const double*>(lv.off);
        it.n_px = n_px;
        it.W = static_cast<unsigned>(lv.w);
        it.first_block = nb;
        it.n_blocks = static_cast<unsigned>((n_px + kMrTile - 1) / kMrTile);
        it.n_fields = static_cast<unsigned>(io.n_fields);
        nb += it.n_blocks;
        it.range = stg.in(io.range, n_px);
        it.poses = stg.in(io.poses, lv.w * 16);
        for (size_t k = 0; k < io.n_fields; ++k) {
            const ob_map_field& fd = io.fields[k];
            it.f[k] = MrField{stg.in(fd.data, n_px * fd.channels * field_bytes(fd.type)), fd.type, fd.channels};
        }
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage map rows inputs");
        hi.push_back(it);
    }
    if (hi.empty()) return OB_OK;
    const unsigned ni = static_cast<unsigned>(hi.size());
    auto* tab = stg.scratch<MrItem>(hi.size());
    auto* b = stg.scratch<uint8_t>(state_bytes(nb) + static_cast<size_t>(nb) * 16 + ni * 8ull);
    double* dout = res.array(rows, cols * 8);
    cudaError_t e = stg.error();
    if (e == cudaSuccess) e = cudaMemcpyAsync(tab, hi.data(), hi.size() * sizeof(MrItem), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(b, 0, state_bytes(nb), st);  // ticket + state words
    if (e != cudaSuccess) return fail_cuda(e, "stage map rows");
    Lookback lb;
    lb.state = reinterpret_cast<uint32_t*>(b + 16);
    lb.agg = reinterpret_cast<unsigned long long*>(b + state_bytes(nb));
    lb.incl = lb.agg + nb;
    unsigned long long* item_end = lb.incl + nb;
    launch(OB_FAM_VOXEL_MAP, map_rows_kernel, nb, kMrThreads, 0, st, tab, ni,
           static_cast<unsigned>(cols), reinterpret_cast<unsigned*>(b), lb, item_end, dout, capacity);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "map rows launch");
    return res.finish(item_end + (ni - 1));
}
