// ob_rows.cuh -- point rows of the C ABI (ob_point_rows) as the device sees them, shared by the voxel map / ICP
// (ob_voxel_map.cu) and cloud-to-cloud ICP (ob_align.cu): a host row count or a device word clamped to the
// capacity, float32 or float64 rows widened to double on load, the order-preserving compaction of the rows an
// association kept, and the host-side check and staging.
#pragma once
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <cstdint>

#include "ob_api_common.h"

namespace ob {
namespace {

// rows of an input: n on the host, or a device word clamped to the capacity
struct Rows {
    const void* p;
    const unsigned long long* n_dev;
    unsigned long long n_host;
    unsigned cap;
};
__device__ __forceinline__ unsigned rows_n(const Rows& r) {
    if (r.n_dev == nullptr) return static_cast<unsigned>(r.n_host);
    const unsigned long long n = *r.n_dev;
    return n < r.cap ? static_cast<unsigned>(n) : r.cap;
}
template <typename T>
__device__ __forceinline__ void load3(const void* base, size_t row, double* v) {
    const T* p = static_cast<const T*>(base) + row * 3;
    v[0] = static_cast<double>(p[0]);
    v[1] = static_cast<double>(p[1]);
    v[2] = static_cast<double>(p[2]);
}

// Order-preserving compaction of the rows i < cap with valid[i] set, one thread per row in blocks of kThreads whose
// flags sum to block_count[b]: keep(i, o) for each such row, o its position among them; the last block writes their
// number to *n.
template <int kThreads, class Keep>
__device__ __forceinline__ void compact_rows(unsigned cap, const uint32_t* valid, const uint32_t* block_count,
                                             unsigned long long* n, Keep keep) {
    using BR = cub::BlockReduce<unsigned, kThreads>;
    using BS = cub::BlockScan<unsigned, kThreads>;
    __shared__ union {
        typename BR::TempStorage r;
        typename BS::TempStorage s;
    } tmp;
    __shared__ unsigned base;
    unsigned part = 0;
    for (unsigned b = threadIdx.x; b < blockIdx.x; b += blockDim.x) part += block_count[b];
    const unsigned before = BR(tmp.r).Sum(part);
    if (threadIdx.x == 0) base = before;
    __syncthreads();
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned f = i < cap ? valid[i] : 0u;
    unsigned pos, total;
    BS(tmp.s).ExclusiveSum(f, pos, total);
    if (f) keep(i, static_cast<size_t>(base) + pos);
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *n = base + total;
}

// ---- host side ----
bool dtype_ok(int32_t d) { return d == OB_F32 || d == OB_F64; }

// rows an input's buffers hold: n, or `capacity` with a device-resident count
size_t row_capacity(size_t n, const void* n_device, size_t capacity) { return n_device ? capacity : n; }

// the count fields of Rows for an input row count (n, or the device word n_device clamped to `capacity`):
// at most 2^31-1 rows per call (else `too_many`), and n_device must be device memory
ob_status count_rows(size_t n, const void* n_device, size_t capacity, Rows* r,
                     const char* too_many = "too many points in one call") {
    const size_t cap = row_capacity(n, n_device, capacity);
    if (cap > 0x7fffffffu) return fail(OB_INVALID_ARGUMENT, too_many);
    if (n_device && !is_device_ptr(n_device)) return fail(OB_INVALID_ARGUMENT, "n_device must be device memory");
    r->n_dev = static_cast<const unsigned long long*>(n_device);
    r->n_host = n;
    r->cap = static_cast<unsigned>(cap);
    return OB_OK;
}

// validate an ob_point_rows and stage it: host rows go through scratch
ob_status stage_rows(const ob_point_rows* in, Staging& stg, Rows* r, const char* what) {
    if (!dtype_ok(in->dtype)) return fail(OB_INVALID_ARGUMENT, "unknown dtype");
    ob_status rs = count_rows(in->n, in->n_device, in->capacity, r);
    if (rs != OB_OK) return rs;
    if (r->cap && !in->points) return fail(OB_INVALID_ARGUMENT, "null points buffer");
    r->p = stg.in(in->points, r->cap * 3ull * (in->dtype == OB_F64 ? 8 : 4));
    if (cudaError_t e = stg.error()) return fail_cuda(e, what);
    return OB_OK;
}

}  // namespace
}  // namespace ob
