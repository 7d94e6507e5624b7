// ob_dewarp_frame.cu -- K3: range image -> world-frame point list in ONE launch:
// LUT projection + per-column pose + range filter + order-preserving compaction.
//
// What it replaces (reference paths relative to /root/reference):
//   dewarp<T>(LidarFrame, XYZLutT<T>, min_range, max_range)  ouster_core/include/ouster/core/pose_util.h:456-485
//   impl::dewarp_impl (single frame)                         ouster_core/include/ouster/core/impl/dewarp_impl.h:22-76
//   dewarp<T>(FrameSet, xyzluts, min_range, max_range)       pose_util.h:475, impl/dewarp_impl.h:84-102
// The reference projects the whole image (cartesian), then walks the columns between the first and
// the last valid one and appends the posed points that pass the range filter; its own note
// (dewarp_impl.h:27-29) asks for the projection to be folded in.  Here nothing is materialised and the
// three passes of a compaction (count, scan, emit) are one kernel:
//   * a CTA owns 32 consecutive columns of one frame (all rows); CTAs take their logical index from a
//     ticket counter, so a CTA's predecessors are always running (or done) when it waits for them;
//   * count : warp = 16-row slab, lane = column: surviving pixels per (slab, column) in shared memory;
//   * scan  : the columns' totals are scanned inside the CTA; the CTA's base comes from a decoupled
//             look-back over its predecessors' published aggregates / inclusive prefixes (one warp looks
//             at 32 predecessors at a time), frames of a set simply continue the chain, so the points of
//             frame f follow those of frame f-1 exactly like the reference's concatenation;
//   * emit  : the count mapping again (the CTA's 16 KB of range are L1 hits): each lane projects its
//             pixel from the LUT, applies the column pose (cast from double to T like the reference) and
//             writes at base + rank (column-major order, rows ascending inside a column -- the order of
//             the reference's loop).
// The number of points is a device-side word (per frame: the inclusive prefix at the frame's last CTA):
// no host round trip sits between the passes.
#include <algorithm>

#include "ob_internal.h"
#include "ob_lookback.cuh"
#include "ob_project.cuh"

namespace ob {

constexpr int kSlabRows = 16;

// Scratch of one launch (zeroed by the launcher): ticket, then per logical CTA a state word
// (0 = nothing yet, 1 = aggregate published, 2 = inclusive prefix published) and the two values.
struct K3Scan {
    unsigned* ticket;
    uint32_t* state;
    unsigned long long* agg;
    unsigned long long* incl;
    unsigned long long* frame_end;  // [n_frames] points up to and including frame f
};

template <typename T>
__global__ void __launch_bounds__(256) k3_fused_kernel(const K3Frame* __restrict__ frames, unsigned n_frames,
                                                       uint32_t min_r, uint32_t max_r, K3Scan sc,
                                                       T* __restrict__ points, uint32_t* __restrict__ frame_idx,
                                                       uint32_t* __restrict__ col_idx, uint64_t* __restrict__ ts_out,
                                                       unsigned long long capacity) {
    extern __shared__ uint32_t s_cnt[];  // [n_slabs][32]
    __shared__ unsigned s_bid;
    __shared__ int s_first, s_last;
    __shared__ unsigned long long s_excl;
    __shared__ uint32_t s_coloff[32];
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5, nw = blockDim.x >> 5;
    if (tid == 0) {
        s_bid = atomicAdd(sc.ticket, 1u);
        s_first = 0x7fffffff;
        s_last = -1;
    }
    __syncthreads();
    const unsigned bid = s_bid;
    unsigned f = 0;
    while (f + 1 < n_frames && frames[f + 1].first_block <= bid) ++f;
    const K3Frame& fr = frames[f];
    const unsigned cg = bid - fr.first_block, W = fr.W, H = fr.H, n_slabs = fr.n_slabs;

    // LidarFrame::get_first_valid_column / get_last_valid_column (lidar_frame.cpp:907-925)
    {
        int lf = 0x7fffffff, ll = -1;
        for (unsigned c = tid; c < W; c += blockDim.x)
            if ((fr.status[c] & 1u) != 0) {
                lf = min(lf, static_cast<int>(c));
                ll = max(ll, static_cast<int>(c));
            }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            lf = min(lf, __shfl_xor_sync(0xffffffffu, lf, d));
            ll = max(ll, __shfl_xor_sync(0xffffffffu, ll, d));
        }
        if (lane == 0) {
            atomicMin(&s_first, lf);
            atomicMax(&s_last, ll);
        }
    }
    // ---- count ----
    const unsigned col = cg * 32u + lane;
    const bool col_ok = col < W;
    for (unsigned slab = warp; slab < n_slabs; slab += nw) {
        const unsigned r0 = slab * kSlabRows, r1 = min(H, r0 + kSlabRows);
        uint32_t c = 0;
        if (col_ok)
            for (unsigned row = r0; row < r1; ++row) {
                const uint32_t r = fr.range[static_cast<size_t>(row) * W + col];
                c += (r >= min_r && r <= max_r) ? 1u : 0u;
            }
        s_cnt[slab * 32u + lane] = c;
    }
    __syncthreads();
    // ---- scan: columns of the CTA, then the look-back over the CTAs before it ----
    if (warp == 0) {
        const int first = s_first, last = s_last;
        // dewarp_impl.h:59-62: columns outside [first, last] are never visited, status == 0 is skipped
        const bool on = col_ok && last >= first && static_cast<int>(col) >= first && static_cast<int>(col) <= last &&
                        fr.status[col] != 0;
        uint32_t mine = 0;
        if (on)
            for (unsigned sl = 0; sl < n_slabs; ++sl) mine += s_cnt[sl * 32u + lane];
        uint32_t incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= static_cast<unsigned>(d)) incl += v;
        }
        s_coloff[lane] = on ? incl - mine : 0xffffffffu;
        const unsigned long long aggregate = __shfl_sync(0xffffffffu, incl, 31);
        const unsigned long long excl = lookback_exclusive(Lookback{sc.state, sc.agg, sc.incl}, bid, aggregate, lane);
        if (lane == 0) {
            s_excl = excl;
            if (cg + 1 == fr.n_cg) sc.frame_end[f] = excl + aggregate;
        }
    }
    __syncthreads();
    // ---- emit ----
    const uint32_t coloff = s_coloff[lane];
    if (coloff == 0xffffffffu) return;
    const unsigned long long cbase = s_excl + coloff;
    const T* dir = static_cast<const T*>(fr.dir);
    const T* off = static_cast<const T*>(fr.off);
    T m[12];  // rows 0..2 of body_to_world[col], cast to T (dewarp_impl.h:64-65)
#pragma unroll
    for (int k = 0; k < 12; ++k) m[k] = static_cast<T>(fr.poses[static_cast<size_t>(col) * 16 + k]);
    const uint64_t ts = (ts_out != nullptr && fr.timestamps != nullptr) ? fr.timestamps[col] : 0ull;
    for (unsigned slab = warp; slab < n_slabs; slab += nw) {
        unsigned long long w = cbase;
        for (unsigned sl = 0; sl < slab; ++sl) w += s_cnt[sl * 32u + lane];
        if (s_cnt[slab * 32u + lane] == 0u) continue;
        const unsigned r0 = slab * kSlabRows, r1 = min(H, r0 + kSlabRows);
        for (unsigned row = r0; row < r1; ++row) {
            const size_t px = static_cast<size_t>(row) * W + col;
            const uint32_t r = fr.range[px];
            if (r >= min_r && r <= max_r) {
                if (w < capacity) {
                    const T x = project(r, dir[px * 3], off[px * 3]);
                    const T y = project(r, dir[px * 3 + 1], off[px * 3 + 1]);
                    const T z = project(r, dir[px * 3 + 2], off[px * 3 + 2]);
                    T* o = points + w * 3;
                    o[0] = pose_row(m, x, y, z);
                    o[1] = pose_row(m + 4, x, y, z);
                    o[2] = pose_row(m + 8, x, y, z);
                    if (frame_idx != nullptr) frame_idx[w] = fr.index;
                    if (col_idx != nullptr) col_idx[w] = col;
                    if (ts_out != nullptr) ts_out[w] = ts;
                }
                ++w;
            }
        }
    }
}

// scratch layout: [ticket + pad : 16 B][state u32 x nb, padded to 8][agg u64 x nb][incl u64 x nb][frame_end u64 x nf]
static size_t k3_state_bytes(unsigned n_blocks) { return 16 + ((static_cast<size_t>(n_blocks) * 4 + 7) & ~static_cast<size_t>(7)); }
size_t dewarp_scan_scratch_bytes(unsigned n_blocks, unsigned n_frames) {
    return k3_state_bytes(n_blocks) + static_cast<size_t>(n_blocks) * 16 + static_cast<size_t>(n_frames) * 8;
}

cudaError_t launch_dewarp_fused(const K3Frame* frames_dev, unsigned n_frames, unsigned n_blocks, unsigned max_slabs,
                                uint32_t min_r, uint32_t max_r, int dtype, void* scratch, void* points,
                                uint32_t* frame_idx, uint32_t* col_idx, uint64_t* ts_out, unsigned long long capacity,
                                const unsigned long long** frame_end_dev, cudaStream_t st) {
    if (frame_end_dev) *frame_end_dev = nullptr;
    if (n_frames == 0 || n_blocks == 0) return cudaSuccess;
    uint8_t* b = static_cast<uint8_t*>(scratch);
    K3Scan sc;
    sc.ticket = reinterpret_cast<unsigned*>(b);
    sc.state = reinterpret_cast<uint32_t*>(b + 16);
    sc.agg = reinterpret_cast<unsigned long long*>(b + k3_state_bytes(n_blocks));
    sc.incl = sc.agg + n_blocks;
    sc.frame_end = sc.incl + n_blocks;
    if (frame_end_dev) *frame_end_dev = sc.frame_end;
    cudaError_t e = cudaMemsetAsync(b, 0, k3_state_bytes(n_blocks), st);  // ticket + state words
    if (e != cudaSuccess) return e;
    const size_t smem = static_cast<size_t>(max_slabs) * 32 * sizeof(uint32_t);  // the caller keeps H <= kDewarpMaxRows
    if (dtype == OB_F64) {
        if (smem > 48u * 1024u) {
            e = cudaFuncSetAttribute(k3_fused_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
            if (e != cudaSuccess) return e;
        }
        launch(OB_FAM_DEWARP, k3_fused_kernel<double>, n_blocks, 256, smem, st, frames_dev, n_frames, min_r, max_r, sc,
               static_cast<double*>(points), frame_idx, col_idx, ts_out, capacity);
    } else {
        if (smem > 48u * 1024u) {
            e = cudaFuncSetAttribute(k3_fused_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
            if (e != cudaSuccess) return e;
        }
        launch(OB_FAM_DEWARP, k3_fused_kernel<float>, n_blocks, 256, smem, st, frames_dev, n_frames, min_r, max_r, sc,
               static_cast<float*>(points), frame_idx, col_idx, ts_out, capacity);
    }
    return cudaGetLastError();
}

}  // namespace ob
