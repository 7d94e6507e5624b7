// ob_decode_pipe.cu -- K2, pipelined: fused lidar-packet field decode -> LidarFrame fields + destaggered
// range + XYZ, as one persistent warp-specialised CTA per SM.
//
// Same work and same results as decode_kernel (ob_decode.cu; it stays as the path for shapes this
// kernel does not take), restructured so that no compute warp ever waits on a global load:
//
//   * warp NCW   (packet producer): one TMA bulk copy per packet into a 2-deep ring of packet stages;
//     a stage is refilled the moment the last compute warp has arrived on its `pk_done` mbarrier.
//     Irregular tiles (dropped / reordered / zero-filled columns) are gathered by this warp's lanes.
//   * warp NCW+1 (LUT producer): the XYZ LUT slices of a tile stream through a 4-deep ring of
//     24 KB slots (a whole 128-row tile), one 2-D TMA tensor copy per table per sub-tile (box = tile
//     columns x RB rows of direction resp. offset; descriptors built on the host, lut_tensor_maps()).
//   * warp NCW+2 (L2 prefetcher): warms L2 with the packets of the tile after next, so that the packet
//     producer's TMA loads are L2 hits even when DRAM is saturated by the output streams.
//   Both producers read the frame-table entry of tile k+1 while tile k is in flight (the table lives
//   in global memory and a dependent chain of L2 round trips under load costs microseconds).
//   * warps 0..NCW-1 (compute): phase A decodes every field of a pixel from registers and stores the
//     row-major images (lane = frame column); phase B projects the ranges with the LUT slice that is
//     already in shared memory (thread = one 16-byte chunk of a row segment: two conflict-free LDS.128,
//     two STG.128) -- only shared-memory loads, ALU and global stores.
//
// Reference behaviour replaced: see ob_decode.cu (parsing.cpp:628-675, lidar_frame.cpp:1422-1528,
// impl/cartesian.h:36-66, impl/lidar_frame_impl.h:733-760).
#include <cuda.h>
#include <cstring>

#include <mutex>
#include <unordered_map>
#include <vector>

#include "ob_api_common.h"
#include "ob_decode_tile.cuh"

namespace ob {

constexpr int kPipeMaxComputeWarps = 24;
constexpr int kPipeStages = 2;    // packet stages
constexpr int kPipeLutSlotsMax = 4;  // LUT ring depth: 4 when it fits the 227 KB, else 3
constexpr int kPipeTileCols = 64;    // widest tile of this kernel

struct PipeParams {
    DecodeParams d;
    const void* lut_maps;  // launch-level LUT descriptors (2 x CUtensorMap) or null
    const void* lut_an;    // launch-level LUT in LUT-free mode: device LutAnalyticT<T> (else null)
    uint32_t ncw;          // compute warps
    uint32_t cpr;          // 16-byte chunks per row segment of a tile (3 * TC * sizeof(T) / 16)
    uint32_t RB;           // rows per LUT sub-tile (= ncw * 32 / cpr)
    uint32_t n_sub;        // sub-tiles per tile (ceil(H / RB))
    uint32_t slot_bytes;   // bytes of one LUT ring slot (direction + offset box)
    uint32_t box_bytes;    // bytes of one table's rows of a sub-tile (lut_ops tensor copies of box_bytes / lut_ops each)
    uint32_t lut_ops;      // tensor copies per table and sub-tile
    uint32_t pk_chunk;     // bytes per bulk copy of a packet (multiple of 16; the last chunk takes the rest)
    uint32_t lut_off;      // byte offsets inside the dynamic shared memory
    uint32_t stage_off;
    uint32_t nl;           // LUT ring slots (3 or 4)
    uint32_t prefetch;     // L2 prefetch distance of the packet tiles (0 = off)
    uint32_t tma_xyz;      // phase B writes its results over the LUT slices and bulk-stores the rows from shared memory
    uint32_t helpers;      // extra warps that only run phase A (0: the third producer-side warp is the L2 prefetcher)
    uint32_t lane_arrive;  // 1: every compute lane arrives on pk_done itself; 0: __syncwarp + one elected arrival per warp
    uint32_t dyn_rows;     // phase A rows handed out through a shared-memory counter (static layouts)
    // store-warp mode (tma_xyz): the XYZ images of a uniformly strided batch as [frame][row][3 * column] tensors,
    // one per return; the frame index of a tile is (its xyz pointer - xyz_base0) / xyz_fs
    const uint8_t* xyz_base0;
    unsigned long long xyz_fs;  // bytes between frames
    alignas(64) CUtensorMap xyz_map[2];
};

__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const void* tmap, int c0, int c1, uint64_t* bar,
                                                 uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
        "[%0], [%1, {%2, %3}], [%4], %5;" ::"r"(smem_u32(smem_dst)),
        "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}


__device__ __forceinline__ void tma_store_3d(const void* tmap, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(tmap), "r"(c0),
                 "r"(c1), "r"(c2), "r"(smem_u32(smem_src))
                 : "memory");
}

#ifdef OB_K2_STREAM_STORES
#define K2_STV(ptr, val) st_stream_vec(ptr, val)
__device__ __forceinline__ void st_stream_vec(float* p, const float4& v) { __stcs(reinterpret_cast<float4*>(p), v); }
__device__ __forceinline__ void st_stream_vec(double* p, const double2& v) { __stcs(reinterpret_cast<double2*>(p), v); }
#else
#define K2_STV(ptr, val) (*reinterpret_cast<V*>(ptr) = (val))
#endif

// explicit shared-memory accesses by 32-bit shared address: the compiler cannot always prove that a
// pointer derived from the stage base is shared memory and then emits generic loads (measured: they were
// the kernel's main long-scoreboard stall)
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ float4 lds_vec(uint32_t a, float4*) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ double2 lds_vec(uint32_t a, double2*) {
    double2 v;
    asm volatile("ld.shared.v2.f64 {%0,%1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(a));
    return v;
}

__device__ __forceinline__ void sts_vec(uint32_t a, const float4& v) {
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts_vec(uint32_t a, const double2& v) {
    asm volatile("st.shared.v2.f64 [%0], {%1,%2};" ::"r"(a), "d"(v.x), "d"(v.y) : "memory");
}
// one thread arrives for `count` participants
__device__ __forceinline__ void mbar_arrive_cnt(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

// per-stage bookkeeping of the pipelined kernel: the column tables of TileCtl plus a copy of the frame's
// table entry (pointers, flags), staged by the packet producer one tile ahead so that the compute warps
// read them from shared memory instead of chasing the global frame table at the start of every tile
struct PipeTileCtl {  // TileCtl for at most kPipeTileCols columns
    int regular;
    int col_src[kPipeTileCols];
    int col_off[kPipeTileCols];
    unsigned char group_fast[16];  // per packet of the tile (eligibility: at most 16 packets per tile)
};
struct PipeCtl {
    PipeTileCtl t;
    DecodeFrame fr;
    uint32_t j0;    // first frame column of the tile
    uint32_t mode;  // XYZ path of the tile: 0 none, 1 LUT ring, 2 LUT-free
    uint32_t row_ctr[2];  // next undecoded row per 32-column group (dynamic row hand-out of phase A)
};

// MAXT: 864 (24 compute + 3 producer-side warps, 72 registers) or 1024 (up to 6 phase-A helper warps, 64 registers)
template <typename T, int MAXT>
__global__ void __launch_bounds__(MAXT, 1)
    decode_pipe_kernel(const __grid_constant__ PipeParams pp) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const DecodeParams& p = pp.d;
    const DecodeLayout& L = p.L;
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int NCW = static_cast<int>(pp.ncw);
    const int NA = NCW + static_cast<int>(pp.helpers);  // warps that run phase A
    constexpr int NS = kPipeStages;
    const unsigned NL = pp.nl;

    // ---- shared memory carve-up ----
    uint64_t* pk_full = reinterpret_cast<uint64_t*>(smem);  // NS
    uint64_t* pk_done = pk_full + NS;                       // NS
    uint64_t* lut_full = pk_done + NS;                      // kPipeLutSlotsMax
    uint64_t* lut_done = lut_full + kPipeLutSlotsMax;       // kPipeLutSlotsMax
    uint64_t* slot_free = lut_done + kPipeLutSlotsMax;      // kPipeLutSlotsMax (store-warp mode: slot read out by the bulk stores)
    PipeCtl* ctl = reinterpret_cast<PipeCtl*>(smem + 128);  // NS entries
    uint8_t* lut0 = smem + pp.lut_off;
    uint8_t* stage0 = smem + pp.stage_off;

    if (tid == 0) {
        for (int s = 0; s < NS; ++s) {
            // every lane arrives for itself (its own generic-proxy writes / reads of the stage control block):
            // no ordering is borrowed from a __syncwarp in front of a single elected arrival
            mbar_init(&pk_full[s], 32);
            // + the store warp, which reads the stage's control block too
            mbar_init(&pk_done[s], (pp.lane_arrive ? NA * 32 : NA) + (pp.tma_xyz ? (pp.lane_arrive ? 32 : 1) : 0));
        }
        for (unsigned s = 0; s < NL; ++s) {
            mbar_init(&lut_full[s], 1);
            mbar_init(&lut_done[s], pp.ncw);
            mbar_init(&slot_free[s], 1);
        }
        mbar_fence_init();
        fence_proxy_async();
    }
    __syncthreads();  // the only CTA-wide barrier

    const unsigned first = blockIdx.x;
    const unsigned n_my = first < p.n_tiles ? (p.n_tiles - first + gridDim.x - 1) / gridDim.x : 0;
    const unsigned n_ret = p.n_returns;
    const unsigned cds = L.channel_data_size;

    auto tile_of = [&](unsigned k, unsigned& f, unsigned& j0) {
        const unsigned t = first + k * gridDim.x;
        f = t / p.tiles_per_frame;
        j0 = (t - f * p.tiles_per_frame) * p.TC;
    };
    const unsigned tc = p.TC;  // every tile is full (eligibility: W % TC == 0)
    // byte offset (inside a stage) of pixel 0 of tile column t
    auto col_offset = [&](unsigned t) -> int {
        const unsigned g = t >> p.cpp_shift;
        return static_cast<int>(g * p.pkt_stride_s + L.packet_header_size + (t - (g << p.cpp_shift)) * L.col_size +
                                L.col_header_size);
    };
    // XYZ path of a frame: evaluated identically by both producers (from the global frame table)
    auto xyz_mode = [&](const DecodeFrame& fr) -> unsigned {
        if (n_ret == 0 || (fr.xyz[0] == nullptr && fr.xyz[1] == nullptr)) return 0u;
        const void* an = fr.lut_dir != nullptr ? fr.lut_an : pp.lut_an;
        if (an != nullptr) return 2u;
        const void* maps = fr.lut_dir != nullptr ? fr.lut_maps : pp.lut_maps;
        return maps != nullptr ? 1u : 0u;
    };

    if (warp == NCW) {
        // =============================== packet producer ===============================
        uint64_t pol_stream = policy_evict_first();
        constexpr unsigned NWORDS = sizeof(DecodeFrame) / 8;
        static_assert(NWORDS <= 64, "frame table entry larger than two words per lane");
        // entry of the NEXT tile, two 8-byte words per lane, loaded one tile ahead
        uint64_t w0 = 0, w1 = 0;
        auto fetch_entry = [&](unsigned k) {
            unsigned f, j0;
            tile_of(k, f, j0);
            const uint64_t* src = reinterpret_cast<const uint64_t*>(&p.frames[f]);
            if (static_cast<unsigned>(lane) < NWORDS) w0 = src[lane];
            if (static_cast<unsigned>(lane) + 32u < NWORDS) w1 = src[lane + 32];
        };
        if (n_my > 0) fetch_entry(0);
        for (unsigned k = 0; k < n_my; ++k) {
            const int s = k % NS;
            if (k >= static_cast<unsigned>(NS)) mbar_wait(&pk_done[s], ((k / NS) - 1) & 1);
            unsigned f, j0;
            tile_of(k, f, j0);
            PipeCtl& pc = ctl[s];
            PipeTileCtl& c = pc.t;
            uint8_t* st = stage0 + static_cast<size_t>(s) * p.stage_bytes;
            // stage the frame's table entry for the compute warps (and for this warp: `fr` below is the copy)
            {
                uint64_t* dst = reinterpret_cast<uint64_t*>(&pc.fr);
                if (static_cast<unsigned>(lane) < NWORDS) dst[lane] = w0;
                if (static_cast<unsigned>(lane) + 32u < NWORDS) dst[lane + 32] = w1;
            }
            __syncwarp();
            if (k + 1 < n_my) fetch_entry(k + 1);  // in flight while this tile is issued and the next wait runs
            const DecodeFrame& fr = pc.fr;
            if (lane == 0) {
                pc.j0 = j0;
                pc.mode = xyz_mode(fr);
                pc.row_ctr[0] = pc.row_ctr[1] = 0u;
            }
            const bool identity = (fr.flags & kFrameIdentityMap) != 0;
            const bool bulk_ok = (fr.flags & kFrameBulkPackets) != 0;
            const unsigned n_groups = tc >> p.cpp_shift;
            if (identity && bulk_ok && (j0 + tc) / L.cpp <= fr.n_slots) {
                if (lane != 0) mbar_arrive(&pk_full[s]);  // this lane's part of the table entry is written
                if (lane == 0) {
                    c.regular = 1;
                    mbar_expect_tx(&pk_full[s], n_groups * L.packet_size);
                    const unsigned slot0 = j0 / L.cpp;
                    for (unsigned g = 0; g < n_groups; ++g) {
                        uint8_t* dstp = st + static_cast<size_t>(g) * p.pkt_stride_s;
                        const uint8_t* srcp = fr.packets + static_cast<size_t>(slot0 + g) * fr.packet_stride;
                        // several copies per packet: a single bulk operation is served at a fraction of what the
                        // SM can pull from DRAM; independent operations overlap
                        for (unsigned o = 0; o < L.packet_size; o += pp.pk_chunk)
                            bulk_g2s_hint(dstp + o, srcp + o, min(pp.pk_chunk, L.packet_size - o), &pk_full[s], pol_stream);
                    }
                }
                continue;
            }
            // ---- irregular tile: per-column bookkeeping, slow groups gathered by the lanes ----
            if (lane == 0) {
                c.regular = 0;
                for (unsigned g = 0; g < n_groups; ++g) {
                    const unsigned jg = j0 + g * L.cpp;
                    bool fast = bulk_ok;
                    int slot = -1;
                    for (unsigned i = 0; i < L.cpp; ++i) {
                        int src;
                        if (identity) {
                            const unsigned sl = (jg + i) / L.cpp;
                            src = sl < fr.n_slots ? static_cast<int>(jg + i) : -1;
                        } else {
                            src = fr.col_src[jg + i];
                        }
                        c.col_src[g * L.cpp + i] = src;
                        c.col_off[g * L.cpp + i] = src < 0 ? -1 : col_offset(g * L.cpp + i);
                        if (src < 0) {
                            fast = false;
                        } else {
                            const int sl = src / static_cast<int>(L.cpp), ci = src - sl * static_cast<int>(L.cpp);
                            if (ci != static_cast<int>(i) || (i > 0 && sl != slot)) fast = false;
                            slot = sl;
                        }
                    }
                    c.group_fast[g] = fast ? 1 : 0;
                }
            }
            __syncwarp();
            uint32_t tx = 0;
            for (unsigned t = 0; t < tc; ++t) {
                const unsigned g = t >> p.cpp_shift;
                if (c.group_fast[g]) {
                    if ((t & (L.cpp - 1)) == 0) tx += L.packet_size;
                    continue;
                }
                const int src = c.col_src[t];
                if (src < 0) continue;
                const int sl = src / static_cast<int>(L.cpp), ci = src - sl * static_cast<int>(L.cpp);
                const uint8_t* gsrc = fr.packets + static_cast<size_t>(sl) * fr.packet_stride + L.packet_header_size +
                                      static_cast<size_t>(ci) * L.col_size;
                uint8_t* dst = st + static_cast<size_t>(g) * p.pkt_stride_s + L.packet_header_size +
                               static_cast<size_t>(t - (g << p.cpp_shift)) * L.col_size;
                // the column plus the 8 bytes a trailing field read may touch (clamped to the packet)
                const size_t col_end = L.packet_header_size + static_cast<size_t>(ci + 1) * L.col_size;
                const size_t extra = min(static_cast<size_t>(8), L.packet_size - col_end);
                const unsigned nbytes = L.col_size + static_cast<unsigned>(extra);
                if ((reinterpret_cast<uintptr_t>(gsrc) & 3u) == 0) {  // layout is word aligned (eligibility)
                    for (unsigned b = lane * 4; b + 4 <= nbytes; b += 128)
                        *reinterpret_cast<uint32_t*>(dst + b) = *reinterpret_cast<const uint32_t*>(gsrc + b);
                    for (unsigned b = (nbytes & ~3u) + lane; b < nbytes; b += 32) dst[b] = gsrc[b];
                } else {
                    for (unsigned b = lane; b < nbytes; b += 32) dst[b] = gsrc[b];
                }
            }
            __syncwarp();
            if (lane != 0) mbar_arrive(&pk_full[s]);  // this lane's gathered bytes and table words are written
            if (lane == 0) {
                mbar_expect_tx(&pk_full[s], tx);  // lane 0's arrival carries the bulk-copy byte count
                for (unsigned g = 0; g < n_groups; ++g) {
                    if (!c.group_fast[g]) continue;
                    const int slot = c.col_src[g * L.cpp] / static_cast<int>(L.cpp);
                    uint8_t* dstp = st + static_cast<size_t>(g) * p.pkt_stride_s;
                    const uint8_t* srcp = fr.packets + static_cast<size_t>(slot) * fr.packet_stride;
                    for (unsigned o = 0; o < L.packet_size; o += pp.pk_chunk)
                        bulk_g2s_hint(dstp + o, srcp + o, min(pp.pk_chunk, L.packet_size - o), &pk_full[s], pol_stream);
                }
            }
        }
        return;
    }

    if (warp == NCW + 1) {
        // =============================== LUT producer ===============================
        if (lane != 0) return;
        const uint64_t pol_keep = policy_evict_last();
        // the few words of the frame entry this warp needs, fetched one tile ahead
        struct Need {
            const void *xyz0, *xyz1, *lut_dir, *lut_maps, *lut_an;
        };
        auto fetch = [&](unsigned k) -> Need {
            unsigned f, j0;
            tile_of(k, f, j0);
            const DecodeFrame& fr = p.frames[f];
            return Need{fr.xyz[0], fr.xyz[1], fr.lut_dir, fr.lut_maps, fr.lut_an};
        };
        Need nx{};
        if (n_my > 0) nx = fetch(0);
        unsigned g = 0;
        for (unsigned k = 0; k < n_my; ++k) {
            unsigned f, j0;
            tile_of(k, f, j0);
            const Need cur = nx;
            if (k + 1 < n_my) nx = fetch(k + 1);
            unsigned mode = 0;
            if (n_ret != 0 && (cur.xyz0 != nullptr || cur.xyz1 != nullptr)) {
                const void* an = cur.lut_dir != nullptr ? cur.lut_an : pp.lut_an;
                const void* maps = cur.lut_dir != nullptr ? cur.lut_maps : pp.lut_maps;
                mode = an != nullptr ? 2u : (maps != nullptr ? 1u : 0u);
            }
            if (mode != 1u) continue;
            const uint8_t* m = static_cast<const uint8_t*>(cur.lut_dir != nullptr ? cur.lut_maps : pp.lut_maps);
            for (unsigned sub = 0; sub < pp.n_sub; ++sub, ++g) {
                const unsigned slot = NL == 4u ? (g & 3u) : g % 3u;
                const unsigned round = NL == 4u ? (g >> 2) : g / 3u;
                if (g >= NL) mbar_wait(pp.tma_xyz ? &slot_free[slot] : &lut_done[slot], (round - 1u) & 1u);
                uint8_t* dst = lut0 + static_cast<size_t>(slot) * pp.slot_bytes;
                mbar_expect_tx(&lut_full[slot], 2u * pp.box_bytes);
                const unsigned op_bytes = pp.box_bytes / pp.lut_ops, op_rows = pp.RB / pp.lut_ops;
                for (unsigned o = 0; o < pp.lut_ops; ++o) {
                    const int y = static_cast<int>(sub * pp.RB + o * op_rows);
                    tma_load_2d_hint(dst + o * op_bytes, m, static_cast<int>(j0 * 3u), y, &lut_full[slot], pol_keep);
                    tma_load_2d_hint(dst + pp.box_bytes + o * op_bytes, m + 128, static_cast<int>(j0 * 3u), y,
                                     &lut_full[slot], pol_keep);
                }
            }
        }
        return;
    }

    if (pp.tma_xyz && warp == NCW + 2) {
        // =============================== store warp ===============================
        // XYZ of the LUT-ring tiles leaves through TMA bulk stores from the slot the compute warps have just
        // overwritten with their results: wait until every compute warp is done with a sub-tile (lut_done), copy
        // its rows out (lane = row, one copy per row and return), and release the slot to the LUT producer when
        // the copies have read it.  Tiles that do not take that path (irregular columns, shifted range fields,
        // one return) only have their slots forwarded.
        const DecodeParams::Plan& q0 = p.plan[p.range_field[0]];
        const DecodeParams::Plan& q1 = p.plan[p.range_field[n_ret > 1 ? 1 : 0]];
        const bool simple_w = (q0.mb | q1.mb | q0.rs | q1.rs) == 0 && q0.d == 0 && q1.d == 0;
        unsigned g = 0;
        for (unsigned k = 0; k < n_my; ++k) {
            const int s = k % NS;
            mbar_wait(&pk_full[s], (k / NS) & 1);
            const PipeCtl& pc = ctl[s];
            const unsigned j0 = pc.j0, mode = pc.mode;
            if (mode == 1u) {
                T* xo0 = static_cast<T*>(pc.fr.xyz[0]);
                T* xo1 = n_ret > 1 ? static_cast<T*>(pc.fr.xyz[1]) : nullptr;
                const bool tma_tile = pc.t.regular != 0 && simple_w && xo0 != nullptr && xo1 != nullptr;
                const int fi = tma_tile ? static_cast<int>((reinterpret_cast<const uint8_t*>(xo0) - pp.xyz_base0) / pp.xyz_fs) : 0;
                for (unsigned sub = 0; sub < pp.n_sub; ++sub, ++g) {
                    const unsigned slot = NL == 4u ? (g & 3u) : g % 3u;
                    const unsigned round = NL == 4u ? (g >> 2) : g / 3u;
                    mbar_wait(&lut_done[slot], round & 1u);
                    if (tma_tile && lane == 0) {
                        // one tensor copy per return: 32 rows x 96 scalars of the slot -> the frame's XYZ image
                        // (rows past H are clipped by the descriptor's bounds)
                        const uint8_t* sl = lut0 + static_cast<size_t>(slot) * pp.slot_bytes;
                        tma_store_3d(&pp.xyz_map[0], sl, static_cast<int>(j0 * 3u), static_cast<int>(sub * pp.RB), fi);
                        tma_store_3d(&pp.xyz_map[1], sl + pp.box_bytes, static_cast<int>(j0 * 3u),
                                     static_cast<int>(sub * pp.RB), fi);
                        bulk_commit();
                        bulk_wait_read<0>();  // the copies have read the slot
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&slot_free[slot]);
                }
            }
            if (pp.lane_arrive) {
                mbar_arrive(&pk_done[s]);
            } else {
                __syncwarp();
                if (lane == 0) mbar_arrive(&pk_done[s]);
            }
        }
        bulk_wait<0>();  // every copy has reached global memory before the CTA retires
        return;
    }

    if (pp.helpers == 0 && warp == NCW + 2) {
        // =============================== L2 prefetcher ===============================
        // paced by the packet stages: when the packets of tile k have landed, warm L2 with those of tile
        // k + pf (pf = 2: its TMA load is issued one tile from now).  Regular tiles only.
        if (lane != 0 || pp.prefetch == 0) return;
        const unsigned pf = pp.prefetch;
        for (unsigned k = 0; k + pf < n_my + pf; ++k) {
            if (k >= pf) {
                const unsigned kk = k - pf;  // pace: tile kk has landed
                mbar_wait(&pk_full[kk % NS], (kk / NS) & 1);
            }
            if (k >= n_my) break;
            if (k < static_cast<unsigned>(NS)) continue;  // the first tiles are loaded directly
            unsigned f, j0;
            tile_of(k, f, j0);
            const DecodeFrame& fr = p.frames[f];
            constexpr uint32_t regular = kFrameIdentityMap | kFrameBulkPackets;
            if ((fr.flags & regular) != regular || (j0 + tc) / L.cpp > fr.n_slots) continue;
            const unsigned slot0 = j0 / L.cpp, n_groups = tc >> p.cpp_shift;
            for (unsigned gi = 0; gi < n_groups; ++gi)
                bulk_prefetch_l2(fr.packets + static_cast<size_t>(slot0 + gi) * fr.packet_stride, L.packet_size);
        }
        return;
    }

    // =================================== compute warps ===================================
    const bool aligned = p.word_aligned != 0;
    constexpr int VN = 16 / sizeof(T);  // scalars per 16-byte chunk
    using V = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
    const DecodeParams::Plan& pl0 = p.plan[p.range_field[0]];
    const DecodeParams::Plan& pl1 = p.plan[p.range_field[n_ret > 1 ? 1 : 0]];
    const bool simple = (pl0.mb | pl1.mb | pl0.rs | pl1.rs) == 0 && pl0.d == 0 && pl1.d == 0;
    const uint32_t ma0 = pl0.ma, ma1 = pl1.ma;
    auto rng = [](const uint32_t* w, const DecodeParams::Plan& pl, bool valid, bool simple_) -> uint32_t {
        const uint32_t a = w[pl.wa] & pl.ma;
        if (simple_) return valid ? a : 0u;
        const uint32_t b = pl.mb ? (w[pl.wa + 1] & pl.mb) : 0u;
        uint32_t v = __funnelshift_r(a, b, pl.rs);
        v = pl.d >= 0 ? (v << pl.d) : (v >> (-pl.d));
        return valid ? v : 0u;
    };
    // helper warps (index >= NCW + 2) take rows of phase A like the compute warps and skip everything else
    const bool helper = warp >= NCW;
    const int aw = helper ? warp - 2 : warp;  // index among the phase-A warps
    unsigned g = 0;  // running LUT sub-tile index (same sequence as the LUT producer)
    for (unsigned k = 0; k < n_my; ++k) {
        const int s = k % NS;
        PipeCtl& pc = ctl[s];
        PipeTileCtl& c = pc.t;
        uint8_t* st = stage0 + static_cast<size_t>(s) * p.stage_bytes;
        // rows rotate over the warps from tile to tile so that H % NCW leftovers even out
        const int wrot = (aw + static_cast<int>((k * 7u) % static_cast<unsigned>(NA))) % NA;

        mbar_wait(&pk_full[s], (k / NS) & 1);
        const DecodeFrame& fr = pc.fr;  // shared-memory copy
        const unsigned j0 = pc.j0, mode = pc.mode;
        const bool regular = c.regular != 0;

        // ---- column headers (timestamp / measurement_id / status) ----
        if (!helper && (fr.timestamp != nullptr || fr.measurement_id != nullptr || fr.status != nullptr)) {
            for (unsigned t = tid; t < tc; t += static_cast<unsigned>(NCW) * 32u) {
                const int co = regular ? col_offset(t) : c.col_off[t];
                uint64_t ts = 0, mid = 0, stt = 0;
                if (co >= 0) {
                    const uint8_t* colp = st + co - L.col_header_size;
                    ts = extract_smem(colp, L.ts, aligned);
                    mid = extract_smem(colp, L.mid, aligned);
                    stt = extract_smem(colp, L.status, aligned);
                }
                if (fr.timestamp) fr.timestamp[j0 + t] = ts;
                if (fr.measurement_id) fr.measurement_id[j0 + t] = static_cast<uint16_t>(mid);
                if (fr.status) fr.status[j0 + t] = static_cast<uint32_t>(stt);
            }
        }

        // ---- phase A: decode the whole tile; lane = frame column, warp = row (strided) ----
        {
        const unsigned rb = 0u, re = L.H;
        const unsigned wfirst = rb + static_cast<unsigned>(wrot);  // first row of this warp's residue class
        for (unsigned cg = 0; (pp.dyn_rows || wfirst < re) && cg * 32 < tc; ++cg) {
            const unsigned t = cg * 32 + lane;
            const int co = regular ? col_offset(t) : c.col_off[t];
            const bool col_valid = co >= 0;
            const uint8_t* px0 = st + (col_valid ? co : col_offset(t));
            const size_t pix0 = static_cast<size_t>(j0) + t;
            if (p.layout_id != 0) {
                uint8_t* outp[kMaxSlots];
#pragma unroll
                for (int i = 0; i < kMaxSlots; ++i)
                    outp[i] = p.slot_field[i] >= 0 ? static_cast<uint8_t*>(fr.fields[p.slot_field[i]]) : nullptr;
                uint32_t* rdp2[2] = {fr.rd[0], fr.rd[1]};
                const unsigned col = static_cast<unsigned>(pix0);
                const unsigned rstep = static_cast<unsigned>(NA);
                const int all = static_output_mode(p, fr);
                if (pp.dyn_rows) {
                    unsigned* ctr = &pc.row_ctr[cg];
                    // dyn_rows 1: every row through the counter; 2: all but the last round of rows are static
                    const unsigned n_static = pp.dyn_rows == 2u && re >= 2u * rstep ? re / rstep - 1u : 0u;
                    const unsigned wrow0 = static_cast<unsigned>(aw);
                    switch (p.layout_id) {
                        case 1: decode_static_tile_dyn<1>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, ctr, wrow0, rstep, n_static, p); break;
                        case 2: decode_static_tile_dyn<2>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, ctr, wrow0, rstep, n_static, p); break;
                        case 3: decode_static_tile_dyn<3>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, ctr, wrow0, rstep, n_static, p); break;
                        case 4: decode_static_tile_dyn<4>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, ctr, wrow0, rstep, n_static, p); break;
                        default: decode_static_tile_dyn<5>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, ctr, wrow0, rstep, n_static, p); break;
                    }
                    continue;
                }
                switch (p.layout_id) {
                    case 1: decode_static_tile<1>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, wfirst, rstep, p); break;
                    case 2: decode_static_tile<2>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, wfirst, rstep, p); break;
                    case 3: decode_static_tile<3>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, wfirst, rstep, p); break;
                    case 4: decode_static_tile<4>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, wfirst, rstep, p); break;
                    default: decode_static_tile<5>(regular, all, px0, col_valid, true, outp, rdp2, col, L.W, re, wfirst, rstep, p); break;
                }
                continue;
            }
            for (unsigned fi = 0; fi < L.n_fields; ++fi) {
                const DecodeField& fd = L.fields[fi];
                uint8_t* out = static_cast<uint8_t*>(fr.fields[fi]);
                const int rr = fd.range_return;
                uint32_t* rdp = rr >= 0 ? fr.rd[rr] : nullptr;
                if (out == nullptr && rdp == nullptr) continue;
                const DecodeParams::Plan& pl = p.plan[fi];
                const uint32_t es = fd.elem_size;
                const int wf = static_cast<int>(wfirst);
                if (pl.fast && es <= 4) {
                    const uint32_t zv = (fd.zero_pattern & 0xffffu) | ((fd.zero_pattern & 0xffffu) << 16);
                    const bool ho = out != nullptr, hr = rdp != nullptr;
                    if (regular) {
                        if (es == 4) decode_rows_dispatch<4, true>(ho, hr, px0, cds, pl, true, zv, true, out, pix0, L.W, re, wf, NA, rdp, p);
                        else if (es == 2) decode_rows_dispatch<2, true>(ho, hr, px0, cds, pl, true, zv, true, out, pix0, L.W, re, wf, NA, rdp, p);
                        else decode_rows_dispatch<1, true>(ho, hr, px0, cds, pl, true, zv, true, out, pix0, L.W, re, wf, NA, rdp, p);
                    } else {
                        if (es == 4) decode_rows_dispatch<4, false>(ho, hr, px0, cds, pl, col_valid, zv, true, out, pix0, L.W, re, wf, NA, rdp, p);
                        else if (es == 2) decode_rows_dispatch<2, false>(ho, hr, px0, cds, pl, col_valid, zv, true, out, pix0, L.W, re, wf, NA, rdp, p);
                        else decode_rows_dispatch<1, false>(ho, hr, px0, cds, pl, col_valid, zv, true, out, pix0, L.W, re, wf, NA, rdp, p);
                    }
                } else {  // wide or unaligned fields: generic 64-bit extraction
                    for (unsigned row = wfirst; row < re; row += NA) {
                        const uint8_t* px = px0 + row * cds;
                        const uint64_t v = !col_valid ? zero_value(fd) : extract_smem(px, fd, aligned);
                        const size_t pix = static_cast<size_t>(row) * L.W + pix0;
                        if (out != nullptr) store_elem(out, pix, es, v);
                        if (rdp != nullptr) {
                            int dcol = static_cast<int>(pix0) + (p.has_shift ? p.shift[row] : 0);
                            dcol = dcol >= static_cast<int>(L.W) ? dcol - static_cast<int>(L.W) : dcol;
                            rdp[static_cast<size_t>(row) * L.W + dcol] = static_cast<uint32_t>(v);
                        }
                    }
                }
            }
        }
        }

        // Phase-B mapping of this thread (chunk q of sub-tile row rsub, the two pixels it touches, their shared
        // addresses).  Derived per tile from an opaque copy of the thread index: kept live across phase A these
        // ~12 loop invariants cost a spill at the kernel's register cap (864 threads -> 72 registers); the
        // reload sat in front of every tile's first LUT wait.
        unsigned tid_b = static_cast<unsigned>(tid);
        asm volatile("" : "+r"(tid_b));
        // phase-B invariants of this thread: chunk q of row (sub-tile row rsub)
        const unsigned rsub = tid_b / pp.cpr;
        const unsigned q = tid_b - rsub * pp.cpr;
        const unsigned e0 = q * VN;
        const unsigned p0 = e0 / 3u;       // first pixel touched by this chunk
        const unsigned k0 = e0 - 3u * p0;  // component of element 0 inside pixel p0
        const unsigned p1 = (p0 + 1 < tc) ? p0 + 1 : p0;
        bool first_px[VN];                 // element e belongs to pixel p0 (else to p1)
    #pragma unroll
        for (int e = 0; e < VN; ++e) first_px[e] = (k0 + e) < 3u;
        // shared addresses of the two pixels' range words inside stage 0, row 0 (regular tiles)
        const uint32_t stage_sa = smem_u32(stage0);
        const uint32_t lut_sa = smem_u32(lut0) + tid_b * 16u;
        const uint32_t coa = static_cast<uint32_t>(col_offset(p0)) + rsub * cds;
        const uint32_t cob = static_cast<uint32_t>(col_offset(p1)) + rsub * cds;
        const uint32_t sub_step = pp.RB * cds;
        // one output chunk: element e = (e-th pixel's range) * dir + off, +0.0 for an empty return
        auto chunk = [&](uint32_t ra, uint32_t rb, const V& dv, const V& ov) -> V {
            const T fa = static_cast<T>(ra), fb = static_cast<T>(rb);
            const T* de = reinterpret_cast<const T*>(&dv);
            const T* oe = reinterpret_cast<const T*>(&ov);
            V outv;
            T* o2 = reinterpret_cast<T*>(&outv);
    #pragma unroll
            for (int e = 0; e < VN; ++e) {
                const bool fa_e = first_px[e];
                const T v = project_nz(fa_e ? fa : fb, de[e], oe[e]);
                o2[e] = (fa_e ? ra : rb) == 0 ? static_cast<T>(0) : v;
            }
            return outv;
        };


        // ---- phase B: XYZ of the tile's sub-tiles from the LUT slices in shared memory.  All of them were
        //      prefetched into the ring while phase A ran (4 slots = a whole 128-row tile), so the waits
        //      below normally fall through ----
        if (mode == 1u && !helper) {
            T* xo0 = static_cast<T*>(fr.xyz[0]);
            T* xo1 = n_ret > 1 ? static_cast<T*>(fr.xyz[1]) : nullptr;
            const size_t ecol = static_cast<size_t>(j0) * 3 + static_cast<size_t>(q) * VN;
            const bool fast_b = regular && simple && xo0 != nullptr && (n_ret < 2 || xo1 != nullptr);
            const size_t row_step = static_cast<size_t>(pp.RB) * L.W * 3;
            T* x0 = xo0 != nullptr ? xo0 + static_cast<size_t>(rsub) * L.W * 3 + ecol : nullptr;
            T* x1 = xo1 != nullptr ? xo1 + static_cast<size_t>(rsub) * L.W * 3 + ecol : nullptr;
            if (x0 != nullptr) __builtin_assume(__isGlobal(x0));
            if (x1 != nullptr) __builtin_assume(__isGlobal(x1));
            if (fast_b && pp.tma_xyz && xo1 != nullptr) {
                // Results leave through TMA: every thread overwrites the direction chunk it has just read with the
                // first return's XYZ and the offset chunk with the second return's (in place, like K1); the store
                // warp bulk-stores the sub-tile's rows (one 384-byte copy per row and return) straight from the slot
                // once every compute warp has arrived on lut_done, and hands the slot back to the LUT producer when
                // the copies have read it.  That takes the 192 STG.128 of a tile -- 3.3 k cycles of the SM's store
                // port (tools/micro/stg_issue.cu) -- out of the compute warps' way.
                const uint32_t sst = stage_sa + static_cast<uint32_t>(s) * p.stage_bytes;
                uint32_t aa0 = sst + coa + pl0.wa * 4u, ab0 = sst + cob + pl0.wa * 4u;
                uint32_t aa1 = sst + coa + pl1.wa * 4u, ab1 = sst + cob + pl1.wa * 4u;
                unsigned row = rsub;
                for (unsigned sub = 0; sub < pp.n_sub; ++sub, ++g, row += pp.RB) {
                    const unsigned slot = NL == 4u ? (g & 3u) : g % 3u;
                    const unsigned round = NL == 4u ? (g >> 2) : g / 3u;
                    mbar_wait(&lut_full[slot], round & 1u);
                    if (row < L.H) {
                        const uint32_t la = lut_sa + slot * pp.slot_bytes;
                        const V dv = lds_vec(la, static_cast<V*>(nullptr));
                        const V ov = lds_vec(la + pp.box_bytes, static_cast<V*>(nullptr));
                        const uint32_t ra0 = lds_u32(aa0) & ma0, rb0 = lds_u32(ab0) & ma0;
                        const uint32_t ra1 = lds_u32(aa1) & ma1, rb1 = lds_u32(ab1) & ma1;
                        sts_vec(la, chunk(ra0, rb0, dv, ov));
                        sts_vec(la + pp.box_bytes, chunk(ra1, rb1, dv, ov));
                    }
                    aa0 += sub_step;
                    ab0 += sub_step;
                    aa1 += sub_step;
                    ab1 += sub_step;
                    fence_proxy_async();  // generic-proxy results -> visible to the store warp's bulk copies
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&lut_done[slot]);
                }
            } else if (fast_b) {
                // lean path (the normal case): running 32-bit shared addresses and running global pointers
                const uint32_t sst = stage_sa + static_cast<uint32_t>(s) * p.stage_bytes;
                uint32_t aa0 = sst + coa + pl0.wa * 4u, ab0 = sst + cob + pl0.wa * 4u;
                uint32_t aa1 = sst + coa + pl1.wa * 4u, ab1 = sst + cob + pl1.wa * 4u;
                unsigned row = rsub;
                unsigned sub = 0;
                // two sub-tiles per step: both slots' waits first, then all shared-memory loads of both, so that the
                // second half's load latency hides behind the first half's arithmetic (one chunk per thread and
                // sub-tile leaves no other independent work between a wait and its stores)
                for (; sub + 2 <= pp.n_sub; sub += 2, g += 2, row += 2 * pp.RB) {
                    const unsigned slot_a = NL == 4u ? (g & 3u) : g % 3u;
                    const unsigned round_a = NL == 4u ? (g >> 2) : g / 3u;
                    const unsigned slot_b = NL == 4u ? ((g + 1) & 3u) : (g + 1) % 3u;
                    const unsigned round_b = NL == 4u ? ((g + 1) >> 2) : (g + 1) / 3u;
                    mbar_wait(&lut_full[slot_a], round_a & 1u);
                    mbar_wait(&lut_full[slot_b], round_b & 1u);
                    const bool on_a = row < L.H, on_b = row + pp.RB < L.H;
                    const uint32_t la = lut_sa + slot_a * pp.slot_bytes, lb = lut_sa + slot_b * pp.slot_bytes;
                    V dva{}, ova{}, dvb{}, ovb{};
                    uint32_t ra0 = 0, rb0 = 0, ra1 = 0, rb1 = 0, rc0 = 0, rd0 = 0, rc1 = 0, rd1 = 0;
                    if (on_a) {
                        dva = lds_vec(la, static_cast<V*>(nullptr));
                        ova = lds_vec(la + pp.box_bytes, static_cast<V*>(nullptr));
                        ra0 = lds_u32(aa0);
                        rb0 = lds_u32(ab0);
                        if (x1 != nullptr) {
                            ra1 = lds_u32(aa1);
                            rb1 = lds_u32(ab1);
                        }
                    }
                    if (on_b) {
                        dvb = lds_vec(lb, static_cast<V*>(nullptr));
                        ovb = lds_vec(lb + pp.box_bytes, static_cast<V*>(nullptr));
                        rc0 = lds_u32(aa0 + sub_step);
                        rd0 = lds_u32(ab0 + sub_step);
                        if (x1 != nullptr) {
                            rc1 = lds_u32(aa1 + sub_step);
                            rd1 = lds_u32(ab1 + sub_step);
                        }
                    }
                    if (on_a) {
                        K2_STV(x0, chunk(ra0 & ma0, rb0 & ma0, dva, ova));
                        if (x1 != nullptr) K2_STV(x1, chunk(ra1 & ma1, rb1 & ma1, dva, ova));
                    }
                    if (on_b) {
                        K2_STV(x0 + row_step, chunk(rc0 & ma0, rd0 & ma0, dvb, ovb));
                        if (x1 != nullptr) K2_STV(x1 + row_step, chunk(rc1 & ma1, rd1 & ma1, dvb, ovb));
                    }
                    aa0 += 2 * sub_step;
                    ab0 += 2 * sub_step;
                    aa1 += 2 * sub_step;
                    ab1 += 2 * sub_step;
                    x0 += 2 * row_step;
                    if (x1 != nullptr) x1 += 2 * row_step;
                    __syncwarp();
                    if (lane == 0) {
                        mbar_arrive(&lut_done[slot_a]);
                        mbar_arrive(&lut_done[slot_b]);
                    }
                }
                for (; sub < pp.n_sub; ++sub, ++g, row += pp.RB) {
                    const unsigned slot = NL == 4u ? (g & 3u) : g % 3u;
                    const unsigned round = NL == 4u ? (g >> 2) : g / 3u;
                    mbar_wait(&lut_full[slot], round & 1u);
                    if (row < L.H) {
                        const uint32_t la = lut_sa + slot * pp.slot_bytes;
                        const V dv = lds_vec(la, static_cast<V*>(nullptr));
                        const V ov = lds_vec(la + pp.box_bytes, static_cast<V*>(nullptr));
                        const uint32_t ra0 = lds_u32(aa0) & ma0, rb0 = lds_u32(ab0) & ma0;
                        K2_STV(x0, chunk(ra0, rb0, dv, ov));
                        if (x1 != nullptr) {
                            const uint32_t ra1 = lds_u32(aa1) & ma1, rb1 = lds_u32(ab1) & ma1;
                            K2_STV(x1, chunk(ra1, rb1, dv, ov));
                        }
                    }
                    aa0 += sub_step;
                    ab0 += sub_step;
                    aa1 += sub_step;
                    ab1 += sub_step;
                    x0 += row_step;
                    if (x1 != nullptr) x1 += row_step;
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&lut_done[slot]);
                }
            } else {
                // general path: irregular tiles (zero-filled / gathered columns), straddling or shifted
                // range fields, a single requested return
                const int co0 = regular ? col_offset(p0) : c.col_off[p0];
                const int co1 = regular ? col_offset(p1) : c.col_off[p1];
                const bool v0 = co0 >= 0, v1 = co1 >= 0;
                const uint8_t* pa = st + (v0 ? co0 : 0);
                const uint8_t* pb = st + (v1 ? co1 : 0);
                for (unsigned sub = 0; sub < pp.n_sub; ++sub, ++g) {
                    const unsigned slot = NL == 4u ? (g & 3u) : g % 3u;
                    const unsigned round = NL == 4u ? (g >> 2) : g / 3u;
                    mbar_wait(&lut_full[slot], round & 1u);
                    const unsigned row = sub * pp.RB + rsub;
                    if (row < L.H) {
                        const uint32_t la = lut_sa + slot * pp.slot_bytes;
                        const V dv = lds_vec(la, static_cast<V*>(nullptr));
                        const V ov = lds_vec(la + pp.box_bytes, static_cast<V*>(nullptr));
                        const uint32_t* wa = reinterpret_cast<const uint32_t*>(pa + static_cast<size_t>(row) * cds);
                        const uint32_t* wb = reinterpret_cast<const uint32_t*>(pb + static_cast<size_t>(row) * cds);
                        if (x0 != nullptr) K2_STV(x0, chunk(rng(wa, pl0, v0, simple), rng(wb, pl0, v1, simple), dv, ov));
                        if (x1 != nullptr) K2_STV(x1, chunk(rng(wa, pl1, v0, simple), rng(wb, pl1, v1, simple), dv, ov));
                    }
                    if (x0 != nullptr) x0 += row_step;
                    if (x1 != nullptr) x1 += row_step;
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&lut_done[slot]);
                }
            }
        }

        // ---- phase B, LUT-free: direction/offset rebuilt from the per-row / per-column tables ----
        if (mode == 2u && !helper) {
            const LutAnalyticT<T>& an =
                *static_cast<const LutAnalyticT<T>*>(fr.lut_dir != nullptr ? fr.lut_an : pp.lut_an);
            const int co0 = regular ? col_offset(p0) : c.col_off[p0];
            const int co1 = regular ? col_offset(p1) : c.col_off[p1];
            const bool v0 = co0 >= 0, v1 = co1 >= 0;
            const uint8_t* pa = st + (v0 ? co0 : 0);
            const uint8_t* pb = st + (v1 ? co1 : 0);
            T* xo0 = static_cast<T*>(fr.xyz[0]);
            T* xo1 = n_ret > 1 ? static_cast<T*>(fr.xyz[1]) : nullptr;
            if (xo0 != nullptr) __builtin_assume(__isGlobal(xo0));
            if (xo1 != nullptr) __builtin_assume(__isGlobal(xo1));
            const size_t ecol = static_cast<size_t>(j0) * 3 + static_cast<size_t>(q) * VN;
            const T cea = __ldg(an.col + 2 * (j0 + p0)), sea = __ldg(an.col + 2 * (j0 + p0) + 1);
            const T ceb = __ldg(an.col + 2 * (j0 + p1)), seb = __ldg(an.col + 2 * (j0 + p1) + 1);
            const T dist = an.dist, b23 = an.b23;
            const T qa0 = cea * an.b03, qa1 = sea * an.b03, qb0 = ceb * an.b03, qb1 = seb * an.b03;
            // extrinsic row of every element of the chunk (component (k0 + e) % 3)
            T mr[VN][4];
#pragma unroll
            for (int e = 0; e < VN; ++e) {
                const unsigned comp = (k0 + e) % 3u;
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    mr[e][i] = comp == 0 ? an.m[i] : (comp == 1 ? an.m[4 + i] : an.m[8 + i]);
            }
            for (unsigned row = rsub; row < L.H; row += pp.RB) {
                const T* rowt = an.row + 4 * static_cast<size_t>(row);
                const T A = __ldg(rowt), B = __ldg(rowt + 1), sa = __ldg(rowt + 2);
                const T da0 = fma(cea, A, -sea * B), da1 = fma(sea, A, cea * B);
                const T db0 = fma(ceb, A, -seb * B), db1 = fma(seb, A, ceb * B);
                const uint32_t* wa = reinterpret_cast<const uint32_t*>(pa + static_cast<size_t>(row) * cds);
                const uint32_t* wb = reinterpret_cast<const uint32_t*>(pb + static_cast<size_t>(row) * cds);
                const size_t eidx = static_cast<size_t>(row) * L.W * 3 + ecol;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    T* xo = r == 0 ? xo0 : xo1;
                    if (xo == nullptr) continue;
                    const DecodeParams::Plan& pl = r == 0 ? pl0 : pl1;
                    const uint32_t ra = rng(wa, pl, v0, simple), rb = rng(wb, pl, v1, simple);
                    const T ta = static_cast<T>(ra) - dist, tb = static_cast<T>(rb) - dist;
                    const T pa0 = fma(da0, ta, qa0), pa1 = fma(da1, ta, qa1), pa2 = fma(sa, ta, b23);
                    const T pb0 = fma(db0, tb, qb0), pb1 = fma(db1, tb, qb1), pb2 = fma(sa, tb, b23);
                    V outv;
                    T* o2 = reinterpret_cast<T*>(&outv);
#pragma unroll
                    for (int e = 0; e < VN; ++e) {
                        const bool fa = first_px[e];
                        const T x0 = fa ? pa0 : pb0, x1 = fa ? pa1 : pb1, x2 = fa ? pa2 : pb2;
                        const T v = fma(mr[e][0], x0, fma(mr[e][1], x1, fma(mr[e][2], x2, mr[e][3])));
                        o2[e] = (fa ? ra : rb) == 0 ? static_cast<T>(0) : v;
                    }
                    *reinterpret_cast<V*>(xo + eidx) = outv;
                }
            }
        }
        if (pp.lane_arrive) {
            mbar_arrive(&pk_done[s]);  // this lane is done with the stage and its control block
        } else {
            __syncwarp();
            if (lane == 0) mbar_arrive(&pk_done[s]);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side: TMA descriptors of a LUT, eligibility, launch
// ---------------------------------------------------------------------------------------------
namespace {

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) != cudaSuccess ||
            qr != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            return nullptr;
        }
        return reinterpret_cast<EncodeTiledFn>(f);
    }();
    return fn;
}

struct MapKey {
    const void* dir;
    uint32_t box_w, box_h;
    bool operator==(const MapKey& o) const { return dir == o.dir && box_w == o.box_w && box_h == o.box_h; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        return std::hash<const void*>()(k.dir) ^ (static_cast<size_t>(k.box_w) * 0x9e3779b97f4a7c15ull) ^
               (static_cast<size_t>(k.box_h) << 17);
    }
};
std::mutex g_map_mx;
std::unordered_map<MapKey, void*, MapKeyHash> g_maps;  // value: device memory holding 2 CUtensorMap (null: failed)

}  // namespace

const void* lut_tensor_maps(const void* dir, const void* off, int dtype, size_t h, size_t w, uint32_t box_w,
                            uint32_t box_h, int device) {
    if (dir == nullptr || off == nullptr || box_w == 0 || box_h == 0) return nullptr;
    std::lock_guard<std::mutex> lk(g_map_mx);
    const MapKey key{dir, box_w, box_h};
    auto it = g_maps.find(key);
    if (it != g_maps.end()) return it->second;
    void* dev = nullptr;
    EncodeTiledFn enc = encode_tiled_fn();
    const size_t es = dtype == OB_F64 ? 8 : 4;
    const bool ok_shape = enc != nullptr && ((reinterpret_cast<uintptr_t>(dir) | reinterpret_cast<uintptr_t>(off)) & 15u) == 0 &&
                          (w * 3 * es) % 16 == 0 && box_w <= 256 && box_h <= 256 && (box_w * es) % 16 == 0;
    if (ok_shape) {
        alignas(64) CUtensorMap maps[2];
        const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(w) * 3, static_cast<cuuint64_t>(h)};
        const cuuint64_t gstr[1] = {static_cast<cuuint64_t>(w) * 3 * es};
        const cuuint32_t box[2] = {box_w, box_h};
        const cuuint32_t estr[2] = {1, 1};
        const CUtensorMapDataType dt = dtype == OB_F64 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
        bool ok = true;
        const void* base[2] = {dir, off};
        for (int i = 0; i < 2 && ok; ++i)
            ok = enc(&maps[i], dt, 2, const_cast<void*>(base[i]), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
        if (ok) {
            DeviceScope on(device);
            if (cudaMalloc(&dev, sizeof(maps)) == cudaSuccess) {
                if (cudaMemcpy(dev, maps, sizeof(maps), cudaMemcpyHostToDevice) != cudaSuccess) {
                    cudaFree(dev);
                    dev = nullptr;
                }
            } else {
                dev = nullptr;
            }
            cudaGetLastError();
        }
    }
    g_maps.emplace(key, dev);
    return dev;
}

void forget_lut_tensor_maps(const void* dir) {
    std::lock_guard<std::mutex> lk(g_map_mx);
    for (auto it = g_maps.begin(); it != g_maps.end();) {
        if (it->first.dir == dir) {
            if (it->second) cudaFree(it->second);
            it = g_maps.erase(it);
        } else {
            ++it;
        }
    }
}

static bool pipe_geometry(const DecodeLayout& L, uint32_t TC, int lut_dtype, uint32_t ncw, uint32_t* cpr, uint32_t* RB) {
    const uint32_t es = lut_dtype == OB_F64 ? 8 : 4;
    if (TC == 0 || TC % 32 != 0 || TC > 64 || L.W % TC != 0) return false;
    const uint32_t c = 3 * TC * es / 16;
    const uint32_t threads = ncw * 32;
    if (c == 0 || threads % c != 0) return false;
    *cpr = c;
    *RB = threads / c;
    return *RB <= 256;
}

// tensor copies per table and sub-tile: the tunable, reduced until it divides the sub-tile's rows
static uint32_t pipe_lut_ops(const Tunables& tn, uint32_t RB) {
    uint32_t n = static_cast<uint32_t>(std::max(1, tn.decode_pipe_lut_split));
    while (n > 1 && RB % n != 0) --n;
    return n;
}

// Launch shape of the pipelined kernel for a packet layout: packets per tile, compute warps per CTA, CTAs per SM.
//   1 CTA/SM : `decode_pipe_warps` (24) compute warps, as many packets per tile as fit a ~68 KB stage pair
//              (at most 64 columns: a LUT row segment is one TMA box), the 72-register build;
//   2 CTAs/SM: half the warps each, stages of at most 28 KB (pair + 48 KB LUT ring < 113 KB), the 64-register build -- for short columns
//              (<= 64-row sensors), whose tiles are too small to amortise the per-tile hand-offs of one
//              CTA: two independent CTAs overlap each other's waits.  Falls back to 1 CTA/SM when a tile
//              would shrink below 32 columns.
void decode_pipe_shape(const DecodeLayout& L, int device, uint32_t* P_out, uint32_t* ncw_out, uint32_t* ctas_out) {
    const Tunables& tn = tunables(device);
    const uint32_t stride = (L.packet_size + 15) & ~15u;
    const uint32_t cpp = std::max<uint32_t>(L.cpp, 1);
    auto fit = [&](uint32_t stage_budget) {  // packets per tile: power of two, one stage within the budget
        uint32_t P = 1;
        if (tn.decode_tile_packets > 0) P = static_cast<uint32_t>(tn.decode_tile_packets);
        else
            while (P * 2 * stride <= stage_budget && P * 2 * cpp <= 64u) P *= 2;
        return std::max<uint32_t>(1, std::min<uint32_t>(P, static_cast<uint32_t>(kMaxTileCols) / cpp));
    };
    // auto: as many CTAs per SM (up to 3) as the layout allows -- a 128-row packet stage pair needs the whole SM.
    // H100 over the sweep shapes (tools/sweep_k2_ctas.py), 3 vs 1 CTA per SM: 32-row single return 9 % faster,
    // 32-row dual 3-5 % and 64-row single 6-8 % slower, 64-row dual and 128-row equal; 4 = 3 (the register file
    // holds three 288-thread CTAs).  Not re-tuned per shape: no rule wins every shape.
    uint32_t ctas = tn.decode_pipe_ctas == 0 ? 3u : static_cast<uint32_t>(tn.decode_pipe_ctas);
    uint32_t ncw = static_cast<uint32_t>(tn.decode_pipe_warps);
    uint32_t P = fit(68u * 1024u);
    for (; ctas > 1; --ctas) {
        const uint32_t n = std::max<uint32_t>(3u, ncw / ctas / 3u * 3u);             // compute warps per CTA
        const uint32_t lut = kPipeLutSlotsMax * 2u * n * 32u * 16u;                   // 4-slot LUT ring
        const uint32_t per_cta = 228u * 1024u / ctas - 1024u;
        if (per_cta < lut + 4096u) continue;
        const uint32_t Pn = fit((per_cta - lut - 2048u) / 2u);
        if ((n + 3u) * 32u * ctas * 64u > 65536u) continue;                           // registers of the 64-register build
        if (Pn * cpp >= 32u && (Pn * cpp) % 32u == 0 && 2u * Pn * stride + lut + 2048u <= per_cta) {
            P = Pn;
            ncw = n;
            break;
        }
    }
    *P_out = P;
    *ncw_out = ncw;
    *ctas_out = ctas;
}

bool decode_pipe_box(const DecodeLayout& L, int device, int lut_dtype, uint32_t* box_w, uint32_t* box_h) {
    const Tunables& tn = tunables(device);
    if (!tn.decode_pipe || L.cpp == 0) return false;
    uint32_t cpr, RB, P, ncw, ctas;
    decode_pipe_shape(L, device, &P, &ncw, &ctas);
    const uint32_t TC = P * L.cpp;
    if (!pipe_geometry(L, TC, lut_dtype, ncw, &cpr, &RB)) return false;
    *box_w = TC * 3;
    *box_h = RB / pipe_lut_ops(tn, RB);
    return true;
}

// dynamic shared memory layout: [mbarriers 128 B][PipeCtl x stages][LUT ring][packet stages][16 B slack]
static size_t pipe_smem_bytes(const DecodeParams& p, uint32_t ncw, uint32_t nl, uint32_t* lut_off, uint32_t* stage_off) {
    size_t off = 128 + static_cast<size_t>(kPipeStages) * sizeof(PipeCtl);
    off = (off + 127) & ~static_cast<size_t>(127);
    *lut_off = static_cast<uint32_t>(off);
    off += static_cast<size_t>(nl) * 2u * (ncw * 32u * 16u);
    *stage_off = static_cast<uint32_t>(off);
    return off + static_cast<size_t>(kPipeStages) * p.stage_bytes + 16;  // + slack for trailing 8-byte field reads
}
// deepest LUT ring that fits: 4 slots hold the LUT of a whole 128-row tile (no refill is ever waited for)
static uint32_t pipe_ring_slots(const DecodeParams& p, uint32_t ncw, uint32_t ctas) {
    uint32_t lo, so;
    // per-CTA budget: 227 KB alone, half of the SM's 228 KB minus the 1 KB the runtime reserves per CTA otherwise
    const size_t budget = ctas >= 2 ? (228u * 1024u / ctas - 1024u) : 227u * 1024u;
    for (uint32_t nl = kPipeLutSlotsMax; nl >= 3; --nl)
        if (pipe_smem_bytes(p, ncw, nl, &lo, &so) <= budget) return nl;
    return 0;
}

bool decode_pipe_eligible(const DecodeParams& p, const DecodeLaunch& a, int device) {
    const DecodeLayout& L = p.L;
    const Tunables& tn = tunables(device);
    if (!p.word_aligned || p.cpp_shift < 0 || L.W % 4 != 0 || (p.TC % L.cpp) != 0) return false;
    if (static_cast<uint64_t>(L.H) * L.W >= (1ull << 30)) return false;
    uint32_t cpr, RB, P, ncw, ctas;
    decode_pipe_shape(L, device, &P, &ncw, &ctas);
    if (P * L.cpp != p.TC) return false;  // make_decode_params(pipe) takes its tile from the same function
    if (!pipe_geometry(L, p.TC, a.lut_dtype, ncw, &cpr, &RB)) return false;
    if (p.TC > static_cast<uint32_t>(kPipeTileCols) || p.TC / L.cpp > 16u) return false;
    if (pipe_ring_slots(p, ncw, ctas) == 0) return false;
    (void)tn;
    // XYZ path: 16-byte aligned rows, 32-bit range plans and TMA descriptors for every LUT in use
    if (p.n_returns > 0) {
        if (!p.vec_ok || !p.plan_ranges_fast) return false;
        if (a.lut_dir != nullptr && a.lut_maps == nullptr && a.lut_an == nullptr) return false;
        if (!a.frame_luts_have_maps) return false;
    }
    return true;
}

cudaError_t launch_decode_pipe(DecodeParams& p, const DecodeLaunch& a, int device, cudaStream_t st) {
    const Tunables& tn = tunables(device);
    PipeParams pp;
    pp.d = p;
    pp.d.stages = kPipeStages;
    pp.lut_maps = a.lut_maps;
    pp.lut_an = a.lut_an;
    uint32_t shape_p, ctas;
    decode_pipe_shape(p.L, device, &shape_p, &pp.ncw, &ctas);
    if (!pipe_geometry(p.L, p.TC, a.lut_dtype, pp.ncw, &pp.cpr, &pp.RB)) return cudaErrorInvalidValue;
    pp.n_sub = (p.L.H + pp.RB - 1) / pp.RB;
    pp.box_bytes = pp.ncw * 32u * 16u;
    pp.slot_bytes = 2u * pp.box_bytes;
    pp.nl = pipe_ring_slots(p, pp.ncw, ctas);
    if (pp.nl == 0) return cudaErrorInvalidValue;
    const size_t smem = pipe_smem_bytes(p, pp.ncw, pp.nl, &pp.lut_off, &pp.stage_off);
    pp.lane_arrive = tn.decode_pipe_lane_arrive ? 1u : 0u;
    pp.tma_xyz = 0;
    pp.xyz_base0 = nullptr;
    pp.xyz_fs = 1;
    std::memset(pp.xyz_map, 0, sizeof(pp.xyz_map));
    if (tn.decode_pipe_tma_xyz && a.xyz_base[0] != nullptr && a.xyz_base[1] != nullptr && p.n_returns == 2 &&
        a.xyz_frame_stride % 16 == 0 && a.n_frames > 0) {
        // the batch's XYZ images as two [frame][row][3 * column] tensors; box = one LUT sub-tile
        EncodeTiledFn enc = encode_tiled_fn();
        const size_t es = a.lut_dtype == OB_F64 ? 8 : 4;
        const cuuint64_t gdim[3] = {static_cast<cuuint64_t>(p.L.W) * 3, p.L.H, a.n_frames};
        const cuuint64_t gstr[2] = {static_cast<cuuint64_t>(p.L.W) * 3 * es, a.xyz_frame_stride};
        const cuuint32_t box[3] = {p.TC * 3, pp.RB, 1};
        const cuuint32_t estr[3] = {1, 1, 1};
        const CUtensorMapDataType dt = a.lut_dtype == OB_F64 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
        bool ok = enc != nullptr && box[0] <= 256 && box[1] <= 256 && (p.L.W * 3 * es) % 16 == 0;
        for (int r = 0; r < 2 && ok; ++r)
            ok = enc(&pp.xyz_map[r], dt, 3, const_cast<void*>(a.xyz_base[r]), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
        if (ok) {
            pp.tma_xyz = 1;
            pp.xyz_base0 = static_cast<const uint8_t*>(a.xyz_base[0]);
            pp.xyz_fs = std::max<unsigned long long>(a.xyz_frame_stride, 1);
        }
    }
    pp.lut_ops = pipe_lut_ops(tn, pp.RB);
    {
        const uint32_t n = static_cast<uint32_t>(std::max(1, tn.decode_pipe_pk_split));
        pp.pk_chunk = std::max<uint32_t>(16u, ((p.L.packet_size + n - 1) / n + 15u) & ~15u);
    }
    // row hand-out of phase A (tools/k2_parts.py): with the fused cloud the fully dynamic form is ~2 % ahead
    // (the hand-out hides behind phase B's waits), decode-only launches are 6 % faster with fixed rows
    pp.dyn_rows = tn.decode_pipe_dyn_rows >= 3
                      ? (a.any_xyz ? 1u : 0u)
                      : static_cast<uint32_t>(std::max(0, tn.decode_pipe_dyn_rows));
    pp.prefetch = static_cast<uint32_t>(std::max(0, std::min(8, tn.decode_pipe_prefetch)));
    // helper warps need the 1024-thread build (64 registers); static pixel layouts only (the plan-driven
    // row loops are not tuned for the lower register cap)
    pp.helpers = p.layout_id != 0 ? static_cast<uint32_t>(std::max(0, std::min(6, tn.decode_pipe_helpers))) : 0u;
    if ((pp.ncw + 2 + pp.helpers) * 32u > 1024u || ctas > 1 || pp.tma_xyz) pp.helpers = 0;
    const int threads = static_cast<int>(pp.ncw + 2 + std::max<uint32_t>(1u, pp.helpers)) * 32;
    const int grid = static_cast<int>(std::min<uint32_t>(p.n_tiles, static_cast<uint32_t>(tn.sm_count) * ctas));
    void (*kern)(PipeParams);
    if (threads > (kPipeMaxComputeWarps + 3) * 32 || ctas > 1)  // 2 CTAs/SM: 2 x 480 threads x 64 registers
        kern = a.lut_dtype == OB_F64 ? decode_pipe_kernel<double, 1024> : decode_pipe_kernel<float, 1024>;
    else
        kern = a.lut_dtype == OB_F64 ? decode_pipe_kernel<double, (kPipeMaxComputeWarps + 3) * 32>
                                     : decode_pipe_kernel<float, (kPipeMaxComputeWarps + 3) * 32>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    launch(OB_FAM_DECODE_PIPE, kern, std::max(grid, 1), threads, smem, st, pp);
    return cudaGetLastError();
}

}  // namespace ob
