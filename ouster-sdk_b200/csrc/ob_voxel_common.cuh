// ob_voxel_common.cuh -- pieces shared by the voxel-grid downsampling (ob_voxel.cu) and the device voxel map
// (ob_voxel_map.cu): the voxel key of a point, its sort decomposition, the first-appearance numbering of the
// voxels of a sorted batch, and the first_n_point distance gate.  Both translation units must key, order and
// gate points identically, so this is the only copy.
#pragma once
#include <cuda/std/tuple>

#include <cstdint>

#include "ob_arith.cuh"

namespace ob {
namespace {

__device__ __forceinline__ unsigned tid_global() { return blockIdx.x * blockDim.x + threadIdx.x; }
inline unsigned blocks_for(unsigned n) { return (n + 255u) / 256u; }

// ---- keys ----
struct VKey {
    uint32_t pad;  // 1: not a point (slot >= n, or a row POINT_NORMAL skips); sorts after every voxel
    int32_t x, y, z;
};
struct VKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, int32_t&, int32_t&, int32_t&> operator()(VKey& k) const {
        return {k.pad, k.x, k.y, k.z};
    }
};
constexpr int kKeyBits = 97;  // x, y, z and the low bit of pad

__device__ __forceinline__ bool same_key(const VKey& a, const VKey& b) {
    return a.pad == b.pad && a.x == b.x && a.y == b.y && a.z == b.z;
}

// first_n_point's rejection test (voxel_hash_map.h:293-296): a kept point q is within the map resolution of p
__device__ __forceinline__ bool within_resolution(double qx, double qy, double qz, double px, double py, double pz,
                                                  double res_sq) {
    return sqn3(sub(qx, px), sub(qy, py), sub(qz, pz)) < res_sq;
}

// ---- first-appearance numbering of the voxels of a sorted batch ----
// opens[seq] = 1 at the sequence position of the first point of every voxel; its inclusive scan in sequence
// order (vrank) numbers the voxels by first appearance, vrank[cap-1] of them.
__global__ void vx_head_kernel(unsigned cap, const VKey* sk, const uint32_t* sseq, uint32_t* opens) {
    const unsigned q = tid_global();
    if (q >= cap) return;
    const VKey k = sk[q];
    opens[sseq[q]] = (k.pad == 0u && (q == 0 || !same_key(k, sk[q - 1]))) ? 1u : 0u;
}

// seg_start[rank - 1] = sorted position of the voxel's first point
__global__ void vx_seg_kernel(unsigned cap, const VKey* sk, const uint32_t* sseq, const uint32_t* vrank, uint32_t* seg_start) {
    const unsigned q = tid_global();
    if (q >= cap) return;
    const VKey k = sk[q];
    if (k.pad == 0u && (q == 0 || !same_key(k, sk[q - 1]))) seg_start[vrank[sseq[q]] - 1] = q;
}

// Equal keys are contiguous after the sort, so "sk[q] == k" is true on [start, end) and false after it: the
// end is found by galloping then bisecting, O(log len) probes instead of a walk over a dense voxel.
__device__ __forceinline__ unsigned segment_end(unsigned start, unsigned cap, const VKey* sk) {
    const VKey k = sk[start];
    unsigned last = start, step = 1, hi = cap;
    for (;;) {
        const unsigned probe = last + step;
        if (probe >= cap || !same_key(sk[probe], k)) {
            hi = min(probe, cap);
            break;
        }
        last = probe;
        step <<= 1;
    }
    while (hi - last > 1) {
        const unsigned mid = last + (hi - last) / 2;
        if (same_key(sk[mid], k)) last = mid;
        else hi = mid;
    }
    return hi;
}

}  // namespace
}  // namespace ob
