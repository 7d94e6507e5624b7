// ob_cloud.cu -- K1: fused range -> XYZ (LUT projection) + per-row destagger rotation,
// batched over frames and returns.  sm_90a.
//
// What it replaces (reference paths relative to /root/reference):
//   impl::cartesianT<T>        ouster_core/include/ouster/core/impl/cartesian.h:36-66
//   destagger_into<T> (2-D/N-D) ouster_core/include/ouster/core/impl/lidar_frame_impl.h:733-811
//   dewarp<T> after the projection (optional, fused)  ouster_core/include/ouster/core/pose_util.h:37-59
//
// Design (HBM-bound streaming kernel, no tensor cores -- there is no contraction here):
//   * persistent CTAs, interleaved tile schedule; a tile = TW consecutive pixels of one row of
//     one frame, all returns.
//   * a ring of S shared-memory stages filled by TMA bulk copies (cp.async.bulk, SASS UBLKCP)
//     tracked by mbarriers: the LUT direction/offset slices and the range slices of the tile.
//     The LUT slices carry an L2 evict_last policy (re-read by every frame), the per-frame
//     streams evict_first.
//   * each thread turns 4 pixels (3 x 128-bit LDS of direction, 3 of offset, one 128-bit LDS
//     of range per return) into 12 coordinates per return and writes them IN PLACE over the
//     direction (return 0) / offset (return 1) slice; __fmul_rn/__fadd_rn keep the reference's
//     un-fused multiply-add rounding so float/double results are bit-identical to the CPU build.
//   * results leave through TMA bulk stores (cp.async.bulk.global.shared::cta): staggered XYZ
//     straight from the in-place buffers; the destaggered range straight from the *input*
//     range slice when the row shift is a multiple of 4 pixels (16-byte aligned rotation),
//     otherwise through a warp-shuffle realignment (lane L takes lane L-1's uint4) and aligned
//     128-bit stores.
#include <algorithm>
#include <cstdio>

#include "ob_internal.h"
#include "ob_project.cuh"
#include "ob_ptx.cuh"

namespace ob {


template <typename T>
struct CloudParams {
    const T* dir;
    const T* off;
    const uint32_t* range;
    T* xyz;
    uint32_t* rd;
    T* xd;
    unsigned long long range_fs, range_rs, xyz_fs, xyz_rs, rd_fs, rd_rs, xd_fs, xd_rs;
    const T* poses;            // optional: n_frames x W x 16 (row-major 4x4 per column), dewarp fused
    unsigned long long poses_fs;
    const T* planes;           // tiled kernel: the same poses as n_frames x 12 planes of W (pose_planes_kernel)
    const LutAnalyticT<T>* an; // LUT-free mode: per-row / per-column tables instead of dir/off (else null)
    int H, W, TW, tiles_per_row, stages;
    int RT, row_blocks;        // rows per work item (1, or Tunables::cloud_pose_rows with poses) and ceil(H / RT)
    int store_lag;             // tiles between a stage's bulk stores and its refill (0 or 1)
    unsigned n_frames, n_tiles, stage_bytes;
    unsigned short shift[kMaxRows];
};

template <typename T>
struct Vec;  // 16-byte vector of T
template <>
struct Vec<float> {
    using type = float4;
    static constexpr int N = 4;
};
template <>
struct Vec<double> {
    using type = double2;
    static constexpr int N = 2;
};

// 12 consecutive T values (4 pixels x 3) via 16-byte shared-memory accesses
template <typename T>
__device__ __forceinline__ void lds12(const T* s, T (&v)[12]) {
    using V = typename Vec<T>::type;
    constexpr int NV = 12 / Vec<T>::N;
    const V* p = reinterpret_cast<const V*>(s);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        V x = p[i];
        const T* e = reinterpret_cast<const T*>(&x);
#pragma unroll
        for (int j = 0; j < Vec<T>::N; ++j) v[i * Vec<T>::N + j] = e[j];
    }
}
template <typename T>
__device__ __forceinline__ void sts12(T* s, const T (&v)[12]) {
    using V = typename Vec<T>::type;
    constexpr int NV = 12 / Vec<T>::N;
    V* p = reinterpret_cast<V*>(s);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        V x;
        T* e = reinterpret_cast<T*>(&x);
#pragma unroll
        for (int j = 0; j < Vec<T>::N; ++j) e[j] = v[i * Vec<T>::N + j];
        p[i] = x;
    }
}

// 4 consecutive T values via 16-byte shared-memory accesses
template <typename T>
__device__ __forceinline__ void lds4(const T* s, T (&v)[4]) {
    using V = typename Vec<T>::type;
    constexpr int NV = 4 / Vec<T>::N;
    const V* p = reinterpret_cast<const V*>(s);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        V x = p[i];
        const T* e = reinterpret_cast<const T*>(&x);
#pragma unroll
        for (int j = 0; j < Vec<T>::N; ++j) v[i * Vec<T>::N + j] = e[j];
    }
}

struct TileCoord {
    unsigned f;
    int row, c0, tw;
};

template <typename T>
__device__ __forceinline__ TileCoord tile_coord(const CloudParams<T>& p, unsigned t) {
    TileCoord tc;
    const unsigned per_frame = static_cast<unsigned>(p.row_blocks) * p.tiles_per_row;
    tc.f = t / per_frame;
    const unsigned rem = t - tc.f * per_frame;
    const unsigned rb = rem / p.tiles_per_row;
    tc.row = static_cast<int>(rb) * p.RT;  // first row of the tile
    tc.c0 = (rem - rb * p.tiles_per_row) * p.TW;
    tc.tw = min(p.TW, p.W - tc.c0);
    return tc;
}

// Warp-specialised: warp 0 is the copy warp -- one thread issues every TMA load and store of the
// CTA and does the tile bookkeeping (integer divisions, expect_tx, store-drain waits) -- while the
// other warps only compute.  The two sides meet through mbarriers: full[s] (bytes of tile k have
// landed in stage s) and done[s] (every compute thread is finished with stage s, results in
// place).  The copy thread's serial work therefore overlaps the compute of the following tiles
// instead of sitting between two __syncthreads of every tile.
//
// POSE: the variant with per-column poses (dewarp fused after the projection).  Work is handed out
// in items of RPI consecutive rows of one column range; a CTA streams the rows of an item through
// the ring while the item's poses sit in shared memory as 12 planes [element][column] (12 bulk copies per
// item out of the plane form a pre-pass makes of the launch's poses: the 4 columns of a thread are then
// one conflict-free 16-byte access per element), so poses cost one L2 read per RPI rows and no
// shared-memory transposition, and the planes are the only pose bytes a CTA holds.
//
// ANALYTIC: the LUT-free variant (SURVEY 8d): nothing of the LUT is loaded; every thread rebuilds the
// beam direction of its 4 pixels from the row's (cos az cos alt, sin az cos alt, sin alt) and the
// columns' (cos enc, sin enc) -- L1-resident tables of a few KB -- and applies the 3x4 extrinsic.
// Results agree with the LUT path to float rounding (<= 1e-5 norm-wise), not bit for bit.
template <typename T, int R, bool POSE, bool ANALYTIC = false>
__global__ void __launch_bounds__(288) cloud_tma_kernel(const __grid_constant__ CloudParams<T> p) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);           // [kMaxStagesK1] loads landed
    uint64_t* done = reinterpret_cast<uint64_t*>(smem + 64);      // [kMaxStagesK1] compute finished
    uint64_t* pose_bar = reinterpret_cast<uint64_t*>(smem + 128);  // pose slice landed
    const unsigned pose_soa_bytes = POSE ? 12u * p.TW * static_cast<unsigned>(sizeof(T)) : 0u;
    T* pose_soa = reinterpret_cast<T*>(smem + 256);
    uint8_t* stage0 = smem + 256 + pose_soa_bytes;

    const int tid = threadIdx.x;
    const int nct = static_cast<int>(blockDim.x) - 32;  // compute threads
    const int ctid = tid - 32;                          // index among them (< 0: copy warp)
    const int S = p.stages;
    const bool need_lut = (p.xyz != nullptr) || (p.xd != nullptr);
    const bool load_lut = need_lut && !ANALYTIC;
    const unsigned lut_bytes_full = 3u * p.TW * sizeof(T);
    const unsigned RPI = POSE ? static_cast<unsigned>(p.RT) : 1u;

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&done[s], static_cast<uint32_t>(nct));
        }
        if (POSE) mbar_init(pose_bar, 1);
        mbar_fence_init();
        fence_proxy_async();
    }
    __syncthreads();  // the only CTA-wide barrier

    // tiles of this CTA: item (first + j * grid), rows 0..RPI-1 of it in order
    const unsigned first = blockIdx.x;
    const unsigned n_items_my = first < p.n_tiles ? (p.n_tiles - first + gridDim.x - 1) / gridDim.x : 0;
    const unsigned n_my = n_items_my * RPI;

    auto coord = [&](unsigned k) {
        TileCoord tc = tile_coord(p, first + (k / RPI) * gridDim.x);
        if (POSE) tc.row += static_cast<int>(k % RPI);
        return tc;
    };

    // =============================== copy warp ===============================
    if (ctid < 0) {
        if (tid != 0) return;
        const uint64_t pol_keep = policy_evict_last(), pol_stream = policy_evict_first();
        auto issue_load = [&](unsigned k) {
            const TileCoord tc = coord(k);
            const int s = k % S;
            uint8_t* st = stage0 + static_cast<size_t>(s) * p.stage_bytes;
            if (tc.row >= p.H) {  // item overhangs the last rows: empty tile
                mbar_expect_tx(&full[s], 0);
                return;
            }
            const size_t px = static_cast<size_t>(tc.row) * p.W + tc.c0;
            const unsigned lut_b = 3u * tc.tw * sizeof(T);
            const unsigned rng_b = 4u * tc.tw;
            mbar_expect_tx(&full[s], (load_lut ? 2u * lut_b : 0u) + R * rng_b);
            if (load_lut) {
                bulk_g2s_hint(st, p.dir + px * 3, lut_b, &full[s], pol_keep);
                bulk_g2s_hint(st + lut_bytes_full, p.off + px * 3, lut_b, &full[s], pol_keep);
            }
#pragma unroll
            for (int r = 0; r < R; ++r) {
                bulk_g2s_hint(st + 2 * lut_bytes_full + r * 4u * p.TW,
                              p.range + tc.f * p.range_fs + r * p.range_rs + px, rng_b, &full[s],
                              pol_stream);
            }
        };
        // pose planes of item i: 12 bulk copies of the tile's columns.  The single plane buffer is free once
        // every compute thread has arrived on done[] of the previous item's last tile (the loop below waits
        // for the tiles in order), and the compute warps wait on pose_bar before the item's first row.
        auto load_planes = [&](unsigned item) {
            const TileCoord tc = tile_coord(p, first + item * gridDim.x);
            const unsigned pb = tc.tw * static_cast<unsigned>(sizeof(T));
            mbar_expect_tx(pose_bar, 12u * pb);
            const T* src = p.planes + static_cast<size_t>(tc.f) * 12u * p.W + tc.c0;
#pragma unroll
            for (int e = 0; e < 12; ++e)
                bulk_g2s_hint(pose_soa + e * p.TW, src + static_cast<size_t>(e) * p.W, pb, pose_bar, pol_keep);
        };
        if (POSE && n_items_my > 0) load_planes(0);
        const unsigned pre = min(n_my, static_cast<unsigned>(S));
        for (unsigned k = 0; k < pre; ++k) issue_load(k);
        const unsigned lag = p.store_lag ? 1u : 0u;
        for (unsigned k = 0; k < n_my; ++k) {
            const int s = k % S;
            const TileCoord tc = coord(k);
            mbar_wait(&done[s], (k / S) & 1);  // results of tile k are in place
            if (POSE && (k % RPI) == RPI - 1 && k + 1 < n_my) load_planes(k / RPI + 1);
            if (tc.row < p.H) {
                uint8_t* st = stage0 + static_cast<size_t>(s) * p.stage_bytes;
                const T* dir_s = reinterpret_cast<const T*>(st);
                const T* off_s = reinterpret_cast<const T*>(st + lut_bytes_full);
                const uint32_t* rng_s = reinterpret_cast<const uint32_t*>(st + 2 * lut_bytes_full);
                const size_t px = static_cast<size_t>(tc.row) * p.W + tc.c0;
                if (p.xyz != nullptr) {
#pragma unroll
                    for (int r = 0; r < R; ++r)
                        bulk_s2g(p.xyz + tc.f * p.xyz_fs + r * p.xyz_rs + px * 3, r == 0 ? dir_s : off_s,
                                 3u * tc.tw * sizeof(T));
                }
                const bool want_d = p.rd != nullptr || p.xd != nullptr;
                const int sh = want_d ? p.shift[tc.row] : 0;
                if ((sh & 3) == 0 && want_d) {  // 16-byte aligned rotation: straight from the stage
                    int d0 = tc.c0 + sh;
                    d0 = d0 >= p.W ? d0 - p.W : d0;
                    const int n1 = min(tc.tw, p.W - d0);
                    const size_t rowpx = static_cast<size_t>(tc.row) * p.W;
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        if (p.rd != nullptr) {
                            uint32_t* drow = p.rd + tc.f * p.rd_fs + r * p.rd_rs + rowpx;
                            const uint32_t* src = rng_s + r * p.TW;
                            bulk_s2g(drow + d0, src, 4u * n1);
                            if (n1 < tc.tw) bulk_s2g(drow, src + n1, 4u * (tc.tw - n1));
                        }
                        if (p.xd != nullptr) {
                            T* drow = p.xd + tc.f * p.xd_fs + r * p.xd_rs + rowpx * 3;
                            const T* src = r == 0 ? dir_s : off_s;
                            bulk_s2g(drow + static_cast<size_t>(d0) * 3, src, 3u * n1 * sizeof(T));
                            if (n1 < tc.tw)
                                bulk_s2g(drow, src + static_cast<size_t>(n1) * 3,
                                         3u * (tc.tw - n1) * sizeof(T));
                        }
                    }
                }
            }
            bulk_commit();  // one group per tile (possibly empty) keeps the wait arithmetic uniform
            // refill a stage whose bulk stores have finished READING smem: lag 0 = this tile's
            // (wait for the stores just issued), lag 1 = the previous tile's (had a tile time to drain)
            if (k >= lag && (k - lag + S) < n_my) {
                if (lag == 0) bulk_wait_read<0>();
                else bulk_wait_read<1>();
                issue_load(k - lag + S);
            }
        }
        bulk_wait<0>();
        return;
    }

    // ============================== compute warps ==============================
    const int lane = tid & 31;
    const int cwarp = ctid >> 5;
    // ring position, its phase, and the position inside the work item are carried along instead of
    // being re-derived from k with integer divisions on every tile
    int s = -1;
    unsigned phase = 1, rr = RPI - 1, item = ~0u;
    TileCoord item_tc{};
    for (unsigned k = 0; k < n_my; ++k) {
        if (++s == S) s = 0;
        if (s == 0) phase ^= 1u;
        if (++rr == RPI) {
            rr = 0;
            ++item;
            item_tc = tile_coord(p, first + item * gridDim.x);
        }
        TileCoord tc = item_tc;
        tc.row += static_cast<int>(rr);
        uint8_t* st = stage0 + static_cast<size_t>(s) * p.stage_bytes;
        T* dir_s = reinterpret_cast<T*>(st);
        T* off_s = reinterpret_cast<T*>(st + lut_bytes_full);
        uint32_t* rng_s = reinterpret_cast<uint32_t*>(st + 2 * lut_bytes_full);

        mbar_wait(&full[s], phase);
        if (POSE && rr == 0) mbar_wait(pose_bar, item & 1u);  // the item's pose planes have landed
        if (POSE && tc.row >= p.H) {
            mbar_arrive(&done[s]);
            continue;
        }

        const int sh = (p.rd != nullptr || p.xd != nullptr) ? p.shift[tc.row] : 0;
        const int q = sh & 3;
        const int n_groups = tc.tw >> 2;

        // ---- destaggered range, unaligned row shift: warp-shuffle realignment ----
        if (p.rd != nullptr && q != 0) {
            const int nv = n_groups;  // source vectors; dest vectors m = 0..nv (edges partial)
            const int base_col = tc.c0 + sh - q;  // multiple of 4
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const uint4* s4 = reinterpret_cast<const uint4*>(rng_s + r * p.TW);
                uint32_t* drow = p.rd + tc.f * p.rd_fs + r * p.rd_rs + static_cast<size_t>(tc.row) * p.W;
                for (int m0 = cwarp * 32; m0 <= nv; m0 += nct) {
                    const int m = m0 + lane;
                    uint4 b = make_uint4(0, 0, 0, 0);
                    if (m < nv) b = s4[m];
                    uint4 a;
                    a.x = __shfl_up_sync(0xffffffffu, b.x, 1);
                    a.y = __shfl_up_sync(0xffffffffu, b.y, 1);
                    a.z = __shfl_up_sync(0xffffffffu, b.z, 1);
                    a.w = __shfl_up_sync(0xffffffffu, b.w, 1);
                    if (lane == 0) a = (m > 0 && m <= nv) ? s4[m - 1] : make_uint4(0, 0, 0, 0);
                    if (m > nv) continue;
                    uint4 o;
                    if (q == 1) o = make_uint4(a.w, b.x, b.y, b.z);
                    else if (q == 2) o = make_uint4(a.z, a.w, b.x, b.y);
                    else o = make_uint4(a.y, a.z, a.w, b.x);
                    int col = base_col + 4 * m;
                    col = col >= p.W ? col - p.W : col;
                    col = col >= p.W ? col - p.W : col;
                    uint32_t* dst = drow + col;
                    if (m == 0) {  // elements e >= q come from this tile
                        const uint32_t ov[4] = {o.x, o.y, o.z, o.w};
                        for (int e = q; e < 4; ++e) stg_stream(dst + e, ov[e]);
                    } else if (m == nv) {  // elements e < q
                        const uint32_t ov[4] = {o.x, o.y, o.z, o.w};
                        for (int e = 0; e < q; ++e) stg_stream(dst + e, ov[e]);
                    } else {
                        stg_stream(reinterpret_cast<uint4*>(dst), o);
                    }
                }
            }
        }

        // ---- LUT-free projection into the (otherwise unused) direction / offset slices ----
        if (ANALYTIC && need_lut && !POSE) {
            using V = typename Vec<T>::type;
            const LutAnalyticT<T>& an = *p.an;
            const T* rowt = an.row + 4 * static_cast<size_t>(tc.row);
            const T A = __ldg(rowt), B = __ldg(rowt + 1), sa = __ldg(rowt + 2);
            const T dist = an.dist, b03 = an.b03, b23 = an.b23;
            T m[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) m[i] = an.m[i];
            for (int g = ctid; g < n_groups; g += nct) {
                T cs[8];  // (cos enc, sin enc) of the 4 columns
                const V* cp = reinterpret_cast<const V*>(an.col + 2 * static_cast<size_t>(tc.c0 + 4 * g));
#pragma unroll
                for (int i = 0; i < 8 / Vec<T>::N; ++i) {
                    const V x = __ldg(cp + i);
                    const T* e = reinterpret_cast<const T*>(&x);
#pragma unroll
                    for (int j = 0; j < Vec<T>::N; ++j) cs[i * Vec<T>::N + j] = e[j];
                }
                uint4 rv4[R];
#pragma unroll
                for (int r = 0; r < R; ++r) rv4[r] = reinterpret_cast<const uint4*>(rng_s + r * p.TW)[g];
                T d0[4], d1[4], q0[4], q1[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const T ce = cs[2 * i], se = cs[2 * i + 1];
                    d0[i] = fma(ce, A, -se * B);
                    d1[i] = fma(se, A, ce * B);
                    q0[i] = ce * b03;
                    q1[i] = se * b03;
                }
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const uint32_t rv[4] = {rv4[r].x, rv4[r].y, rv4[r].z, rv4[r].w};
                    T out[12];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const T t = static_cast<T>(rv[i]) - dist;
                        const T p0 = fma(d0[i], t, q0[i]), p1 = fma(d1[i], t, q1[i]), p2 = fma(sa, t, b23);
#pragma unroll
                        for (int j = 0; j < 3; ++j) {
                            const T v = fma(m[4 * j], p0, fma(m[4 * j + 1], p1, fma(m[4 * j + 2], p2, m[4 * j + 3])));
                            out[3 * i + j] = rv[i] == 0 ? static_cast<T>(0) : v;
                        }
                    }
                    sts12((r == 0 ? dir_s : off_s) + 12 * g, out);
                }
            }
        }

        // ---- projection (and pose), in place ----
        if (!ANALYTIC && need_lut && !POSE) {
            for (int g = ctid; g < n_groups; g += nct) {
                T d[12], o[12];
                lds12(dir_s + 12 * g, d);
                lds12(off_s + 12 * g, o);
                uint4 rv4[R];
#pragma unroll
                for (int r = 0; r < R; ++r) rv4[r] = reinterpret_cast<const uint4*>(rng_s + r * p.TW)[g];
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const uint32_t rv[4] = {rv4[r].x, rv4[r].y, rv4[r].z, rv4[r].w};
                    T out[12];
#pragma unroll
                    for (int i = 0; i < 12; ++i) out[i] = project(rv[i / 3], d[i], o[i]);
                    sts12((r == 0 ? dir_s : off_s) + 12 * g, out);
                }
            }
        }
        if (need_lut && POSE) {
            // 4 pixels per thread, like the plain path: 16-byte accesses of the LUT slices, the range words and
            // the pose planes (plane e holds element e of the tile's column poses, so the 4 columns of a thread
            // are one conflict-free vector).  One pose row (4 planes) is live at a time to keep the register
            // count of the plain path's occupancy.
            for (int g = ctid; g < n_groups; g += nct) {
                T pt[R][12];  // projected points, sensor frame
                {
                    T d[12], o[12];
                    lds12(dir_s + 12 * g, d);
                    lds12(off_s + 12 * g, o);
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        const uint4 rv4 = reinterpret_cast<const uint4*>(rng_s + r * p.TW)[g];
                        const uint32_t rv[4] = {rv4.x, rv4.y, rv4.z, rv4.w};
#pragma unroll
                        for (int i = 0; i < 12; ++i) pt[r][i] = project(rv[i / 3], d[i], o[i]);
                    }
                }
                T out[R][12];
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    T m0[4], m1[4], m2[4], m3[4];
                    lds4(pose_soa + (4 * j + 0) * p.TW + 4 * g, m0);
                    lds4(pose_soa + (4 * j + 1) * p.TW + 4 * g, m1);
                    lds4(pose_soa + (4 * j + 2) * p.TW + 4 * g, m2);
                    lds4(pose_soa + (4 * j + 3) * p.TW + 4 * g, m3);
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const T mm[4] = {m0[i], m1[i], m2[i], m3[i]};
                            out[r][3 * i + j] = pose_row(mm, pt[r][3 * i], pt[r][3 * i + 1], pt[r][3 * i + 2]);
                        }
                }
#pragma unroll
                for (int r = 0; r < R; ++r) sts12((r == 0 ? dir_s : off_s) + 12 * g, out[r]);
            }
        }

        // ---- destaggered XYZ, unaligned row shift: coalesced 32-bit word copies ----
        if (p.xd != nullptr && q != 0) {
            named_barrier_sync(1, nct);  // every compute thread's results are in the stage
            constexpr int WPE = sizeof(T) / 4;  // 32-bit words per scalar
            const int row_words = p.W * 3 * WPE;
            const int n_words = tc.tw * 3 * WPE;
            int d0 = tc.c0 + sh;
            d0 = d0 >= p.W ? d0 - p.W : d0;
            const int dst0 = d0 * 3 * WPE;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                uint32_t* drow = reinterpret_cast<uint32_t*>(
                    p.xd + tc.f * p.xd_fs + r * p.xd_rs + static_cast<size_t>(tc.row) * p.W * 3);
                const uint32_t* src = reinterpret_cast<const uint32_t*>(r == 0 ? dir_s : off_s);
                for (int i = ctid; i < n_words; i += nct) {
                    int dw = dst0 + i;
                    dw = dw >= row_words ? dw - row_words : dw;
                    stg_stream(drow + dw, src[i]);
                }
            }
        }
        if (need_lut) fence_proxy_async();  // generic-proxy results -> visible to the TMA stores
        mbar_arrive(&done[s]);
    }
}

// Pre-pass of the pose-fused variant: poses [frame][column][16] -> planes [frame][element 0..11][column]
// (rows 0..2 of every 4x4), so that the tiled kernel bulk-copies an item's planes straight into shared
// memory.  64 bytes in, 48 bytes out per column: < 1 % of the launch's traffic.
template <typename T>
__global__ void __launch_bounds__(256) pose_planes_kernel(const T* __restrict__ poses, unsigned long long poses_fs,
                                                          T* __restrict__ planes, unsigned W, unsigned n_frames) {
    const unsigned f = blockIdx.y;
    const unsigned col = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames || col >= W) return;
    using V = typename Vec<T>::type;
    const V* src = reinterpret_cast<const V*>(poses + f * poses_fs + static_cast<size_t>(col) * 16);
    T* dst = planes + static_cast<size_t>(f) * 12u * W + col;
    constexpr int NV = 12 / Vec<T>::N;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const V x = __ldg(src + i);
        const T* e = reinterpret_cast<const T*>(&x);
#pragma unroll
        for (int j = 0; j < Vec<T>::N; ++j) dst[static_cast<size_t>(i * Vec<T>::N + j) * W] = e[j];
    }
}

// Generic kernel: any width / alignment / stride.  One pixel per thread, grid-stride.
template <typename T>
__global__ void cloud_generic_kernel(const __grid_constant__ CloudParams<T> p, int n_returns) {
    const size_t n_px = static_cast<size_t>(p.H) * p.W;
    const size_t total = n_px * p.n_frames;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t f = i / n_px;
        const size_t px = i - f * n_px;
        const int row = static_cast<int>(px / p.W);
        const int col = static_cast<int>(px - static_cast<size_t>(row) * p.W);
        int dcol = col;
        if (p.rd != nullptr || p.xd != nullptr) {
            dcol = col + p.shift[row];
            dcol = dcol >= p.W ? dcol - p.W : dcol;
        }
        const size_t dpx = static_cast<size_t>(row) * p.W + dcol;
        T d[3] = {0, 0, 0}, o[3] = {0, 0, 0};
        if (p.xyz != nullptr || p.xd != nullptr) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                d[c] = p.dir[px * 3 + c];
                o[c] = p.off[px * 3 + c];
            }
        }
        for (int r = 0; r < n_returns; ++r) {
            const uint32_t rv = p.range[f * p.range_fs + r * p.range_rs + px];
            if (p.rd != nullptr) p.rd[f * p.rd_fs + r * p.rd_rs + dpx] = rv;
            if (p.xyz != nullptr || p.xd != nullptr) {
                T v[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) v[c] = project(rv, d[c], o[c]);
                if (p.poses != nullptr) {
                    const T* m = p.poses + f * p.poses_fs + static_cast<size_t>(col) * 16;
                    const T x = v[0], y = v[1], z = v[2];
                    v[0] = pose_row(m, x, y, z);
                    v[1] = pose_row(m + 4, x, y, z);
                    v[2] = pose_row(m + 8, x, y, z);
                }
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    if (p.xyz != nullptr) p.xyz[f * p.xyz_fs + r * p.xyz_rs + px * 3 + c] = v[c];
                    if (p.xd != nullptr) p.xd[f * p.xd_fs + r * p.xd_rs + dpx * 3 + c] = v[c];
                }
            }
        }
    }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <typename T>
cudaError_t launch_cloud(const CloudArgs<T>& a, int device, cudaStream_t st) {
    const Tunables& tn = tunables(device);
    CloudParams<T> p;
    p.dir = a.dir;
    p.off = a.off;
    p.range = a.range;
    p.xyz = a.xyz;
    p.rd = a.rd;
    p.xd = a.xd;
    p.range_fs = a.range_fs;
    p.range_rs = a.range_rs;
    p.xyz_fs = a.xyz_fs;
    p.xyz_rs = a.xyz_rs;
    p.rd_fs = a.rd_fs;
    p.rd_rs = a.rd_rs;
    p.xd_fs = a.xd_fs;
    p.xd_rs = a.xd_rs;
    p.H = a.H;
    p.W = a.W;
    p.n_frames = a.n_frames;
    for (int i = 0; i < kMaxRows; ++i) p.shift[i] = 0;
    if (a.shift != nullptr)
        for (int i = 0; i < a.H && i < kMaxRows; ++i) p.shift[i] = a.shift[i];

    const bool need_lut = a.xyz != nullptr || a.xd != nullptr;
    // element-stride alignment so that every tile slice is 16-byte aligned
    const size_t t4 = 16 / sizeof(T);  // T elements per 16 bytes
    bool fast = !tn.force_generic && (a.W % 4 == 0) && a.H <= kMaxRows && aligned16(a.range) &&
                a.range_fs % 4 == 0 && a.range_rs % 4 == 0;
    const bool analytic = a.analytic != nullptr && need_lut && a.poses == nullptr;
    if (need_lut && !analytic) fast = fast && aligned16(a.dir) && aligned16(a.off);
    if (a.xyz) fast = fast && aligned16(a.xyz) && a.xyz_fs % t4 == 0 && a.xyz_rs % t4 == 0;
    if (a.rd) fast = fast && aligned16(a.rd) && a.rd_fs % 4 == 0 && a.rd_rs % 4 == 0;
    if (a.xd) fast = fast && aligned16(a.xd) && a.xd_fs % t4 == 0 && a.xd_rs % t4 == 0;
    if (a.n_returns < 1 || a.n_returns > 2) return cudaErrorInvalidValue;
    if ((a.rd != nullptr || a.xd != nullptr) && a.H > kMaxRows) return cudaErrorInvalidValue;

    if (a.poses) fast = fast && aligned16(a.poses) && a.poses_fs % t4 == 0;
    p.poses = a.poses;
    p.poses_fs = a.poses_fs;
    p.planes = nullptr;
    p.an = a.analytic;
    p.store_lag = 0;
    p.RT = 1;
    p.row_blocks = a.H;

    if (!fast) {
        p.TW = 0;
        p.tiles_per_row = 0;
        p.stages = 0;
        p.n_tiles = 0;
        p.stage_bytes = 0;
        const size_t total = static_cast<size_t>(a.H) * a.W * a.n_frames;
        const int threads = 256;
        const size_t want = (total + threads - 1) / threads;
        const int blocks = static_cast<int>(std::min<size_t>(want, static_cast<size_t>(tn.sm_count) * 16));
        launch(OB_FAM_CLOUD, cloud_generic_kernel<T>, std::max(blocks, 1), threads, 0, st, p, a.n_returns);
        return cudaGetLastError();
    }

    const bool pose = a.poses != nullptr && need_lut;
    // Single-return frames move half the bytes per tile, so the per-tile fixed cost (mbarrier hand-offs,
    // TMA issue) weighs twice as much: 1024-pixel tiles, 4 stages, 2 CTAs per SM (on H100 every geometry near
    // this one runs within 1 % of the DRAM-bound best, tools/sweep_k1_single.py).
    // (rows of at least 1024 pixels: a 512-wide row is one 512-pixel tile either way)
    const bool wide = tn.cloud_auto && !pose && a.n_returns == 1 && sizeof(T) == 4 && a.W >= 1024;
    int TW = pose ? tn.cloud_pose_tw : (wide ? 1024 : tn.cloud_tw);
    if (sizeof(T) == 8) TW = std::max(4, TW / 2 / 4 * 4);
    TW = std::min(TW, a.W);
    TW = std::max(4, TW / 4 * 4);
    const int RT = pose ? std::min(tn.cloud_pose_rows, std::max(4, a.H)) : 1;
    const int row_blocks = (a.H + RT - 1) / RT;
    // small launches: shrink tiles until every SM has work for a few CTAs
    const unsigned want_tiles = static_cast<unsigned>(tn.sm_count) * tn.cloud_ctas_per_sm * 2;
    while (TW > 128 && static_cast<unsigned>(row_blocks) * ((a.W + TW - 1) / TW) * a.n_frames < want_tiles)
        TW = std::max(128, TW / 2 / 4 * 4);
    p.TW = TW;
    p.RT = RT;
    p.row_blocks = row_blocks;
    p.tiles_per_row = (a.W + TW - 1) / TW;
    p.stages = pose ? tn.cloud_pose_stages : (wide ? 4 : tn.cloud_stages);
    p.store_lag = tn.cloud_store_lag ? 1 : 0;
    if (pose) p.stages = std::max(2, std::min(p.stages, RT - 1));  // the pose double buffer relies on RPI > stages
    p.n_tiles = static_cast<unsigned>(row_blocks) * p.tiles_per_row * a.n_frames;  // work items
    p.stage_bytes = 2u * 3u * TW * sizeof(T) + static_cast<unsigned>(a.n_returns) * 4u * TW;
    p.stage_bytes = (p.stage_bytes + 127u) & ~127u;
    const size_t pose_bytes = pose ? 12u * TW * sizeof(T) : 0u;  // the item's 12 pose planes
    if (p.stages > 8) p.stages = 8;  // barrier arrays hold 8 entries each
    const size_t smem = 256 + pose_bytes + static_cast<size_t>(p.stages) * p.stage_bytes;
    if (smem > 227u * 1024u) return cudaErrorInvalidValue;
    const int ctas = std::max<int>(
        1, std::min<size_t>(pose ? tn.cloud_pose_ctas_per_sm : (wide ? 2 : tn.cloud_ctas_per_sm), (227u * 1024u) / smem));
    const int grid =
        static_cast<int>(std::min<unsigned>(p.n_tiles, static_cast<unsigned>(tn.sm_count) * ctas));
    void (*kern)(CloudParams<T>);
    if (pose) kern = a.n_returns == 2 ? cloud_tma_kernel<T, 2, true> : cloud_tma_kernel<T, 1, true>;
    else if (analytic) kern = a.n_returns == 2 ? cloud_tma_kernel<T, 2, false, true> : cloud_tma_kernel<T, 1, false, true>;
    else kern = a.n_returns == 2 ? cloud_tma_kernel<T, 2, false> : cloud_tma_kernel<T, 1, false>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    T* planes = nullptr;
    if (pose) {  // stream-ordered scratch: the launch's poses as planes
        if (a.n_frames > 65535) return cudaErrorInvalidValue;
        e = cudaMallocAsync(reinterpret_cast<void**>(&planes), static_cast<size_t>(a.n_frames) * 12u * a.W * sizeof(T), st);
        if (e != cudaSuccess) return e;
        launch(OB_FAM_CLOUD, pose_planes_kernel<T>, dim3((a.W + 255) / 256, a.n_frames), 256, 0, st, a.poses,
               a.poses_fs, planes, a.W, a.n_frames);
        p.planes = planes;
    }
    const int threads = (pose ? tn.cloud_pose_threads : tn.cloud_threads) + 32;  // + the copy warp
    launch(OB_FAM_CLOUD, kern, std::max(grid, 1), threads, smem, st, p);
    e = cudaGetLastError();
    if (planes != nullptr) {
        const cudaError_t e2 = cudaFreeAsync(planes, st);
        if (e == cudaSuccess) e = e2;
    }
    return e;
}

// ---------------------------------------------------------------------------------------------
// dewarp / transform: out[i*W + w] = R_w * p[i*W + w] + t_w  (pose_util.h:37-59, 118-131).
// A CTA stages the 3x4 parts of 128 consecutive column poses in shared memory and sweeps a band of
// rows; lane = column, so point loads/stores are contiguous 384-byte runs per warp.
// Each row is ob_project.cuh's pose_row: products rounded separately, summed as x0 + (x1 + x2), then + t.
// ---------------------------------------------------------------------------------------------

template <typename T>
__global__ void __launch_bounds__(256) dewarp_kernel(const T* __restrict__ pts, const T* __restrict__ poses,
                                                     T* __restrict__ out, unsigned long long H,
                                                     unsigned long long W, unsigned rows_per_block) {
    __shared__ T sp[128 * 12];
    const unsigned long long c0 = static_cast<unsigned long long>(blockIdx.x) * 128ull;
    const unsigned ncol = static_cast<unsigned>(min(128ull, W - c0));
    for (unsigned i = threadIdx.x; i < ncol * 12u; i += blockDim.x)
        sp[i] = poses[(c0 + i / 12u) * 16ull + (i % 12u)];
    __syncthreads();
    const unsigned lc = threadIdx.x & 127u;          // column inside the block
    const unsigned rsub = threadIdx.x >> 7;           // 2 rows in flight per 256 threads
    if (lc >= ncol) return;
    const T* m = sp + lc * 12u;
    const unsigned long long r0 = static_cast<unsigned long long>(blockIdx.y) * rows_per_block;
    const unsigned long long r1 = min(H, r0 + rows_per_block);
    for (unsigned long long row = r0 + rsub; row < r1; row += 2) {
        const unsigned long long ix = (row * W + c0 + lc) * 3ull;
        const T x = pts[ix], y = pts[ix + 1], z = pts[ix + 2];
        out[ix] = pose_row(m, x, y, z);
        out[ix + 1] = pose_row(m + 4, x, y, z);
        out[ix + 2] = pose_row(m + 8, x, y, z);
    }
}

template <typename T>
cudaError_t launch_dewarp(const T* pts, const T* poses, T* out, size_t H, size_t W, cudaStream_t st) {
    if (H == 0 || W == 0) return cudaSuccess;
    const unsigned col_blocks = static_cast<unsigned>((W + 127) / 128);
    // enough row bands to fill the machine, at least 8 rows each
    unsigned bands = static_cast<unsigned>(std::max<size_t>(1, std::min<size_t>(H / 8 + 1, 2368 / std::max(1u, col_blocks) + 1)));
    unsigned rows_per_block = static_cast<unsigned>((H + bands - 1) / bands);
    bands = static_cast<unsigned>((H + rows_per_block - 1) / rows_per_block);
    if (bands > 65535) return cudaErrorInvalidValue;
    dim3 grid(col_blocks, bands);
    launch(OB_FAM_DEWARP, dewarp_kernel<T>, grid, 256, 0, st, pts, poses, out, H, W, rows_per_block);
    return cudaGetLastError();
}
template cudaError_t launch_dewarp<float>(const float*, const float*, float*, size_t, size_t, cudaStream_t);
template cudaError_t launch_dewarp<double>(const double*, const double*, double*, size_t, size_t, cudaStream_t);

template cudaError_t launch_cloud<float>(const CloudArgs<float>&, int, cudaStream_t);
template cudaError_t launch_cloud<double>(const CloudArgs<double>&, int, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// Generic destagger (any element size / trailing dims): byte rotation of every row.
// out_row[b] = in_row[(b - shift_bytes) mod row_bytes]; 16-byte aligned stores on the destination,
// source words realigned with a byte funnel shift.
// replaces destagger_into<T> / <T,ndim>  impl/lidar_frame_impl.h:733-811
// ---------------------------------------------------------------------------------------------
struct DestaggerParams {
    const uint8_t* in;
    uint8_t* out;
    unsigned long long row_bytes;
    unsigned px_bytes;
    int H;
    unsigned short shift[kMaxRows];
};

__global__ void destagger_words_kernel(const __grid_constant__ DestaggerParams p) {
    // row_bytes % 4 == 0, base pointers 4-byte aligned
    const unsigned row_words = static_cast<unsigned>(p.row_bytes >> 2);
    const int row = blockIdx.y;
    const unsigned sb = static_cast<unsigned>(p.shift[row]) * p.px_bytes;  // < row_bytes
    const uint32_t* in = reinterpret_cast<const uint32_t*>(p.in + row * p.row_bytes);
    uint32_t* out = reinterpret_cast<uint32_t*>(p.out + row * p.row_bytes);
    const unsigned bsh = (sb & 3u) * 8u;
    for (unsigned dw = blockIdx.x * blockDim.x + threadIdx.x; dw < row_words;
         dw += gridDim.x * blockDim.x) {
        // source byte address of destination byte 4*dw
        long long src = static_cast<long long>(dw) * 4 - sb;
        if (src < 0) src += static_cast<long long>(p.row_bytes);
        unsigned sw = static_cast<unsigned>(src >> 2);
        if (bsh == 0) {
            out[dw] = in[sw];
        } else {
            // src is not word aligned: bytes come from words sw and sw+1 (mod row)
            const unsigned sw1 = (sw + 1 == row_words) ? 0u : sw + 1;
            out[dw] = __funnelshift_r(in[sw], in[sw1], (static_cast<unsigned>(src) & 3u) * 8u);
        }
    }
}

__global__ void destagger_bytes_kernel(const __grid_constant__ DestaggerParams p) {
    const int row = blockIdx.y;
    const unsigned long long sb = static_cast<unsigned long long>(p.shift[row]) * p.px_bytes;
    const uint8_t* in = p.in + row * p.row_bytes;
    uint8_t* out = p.out + row * p.row_bytes;
    for (unsigned long long b = blockIdx.x * blockDim.x + threadIdx.x; b < p.row_bytes;
         b += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        unsigned long long src = b >= sb ? b - sb : b + p.row_bytes - sb;
        out[b] = in[src];
    }
}

// rows beyond kMaxRows: shifts fetched from device memory
__global__ void destagger_bytes_dev_kernel(const uint8_t* in_, uint8_t* out_,
                                           unsigned long long row_bytes, unsigned px_bytes,
                                           const unsigned short* shift) {
    const int row = blockIdx.y;
    const unsigned long long sb = static_cast<unsigned long long>(shift[row]) * px_bytes;
    const uint8_t* in = in_ + row * row_bytes;
    uint8_t* out = out_ + row * row_bytes;
    for (unsigned long long b = blockIdx.x * blockDim.x + threadIdx.x; b < row_bytes;
         b += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        unsigned long long src = b >= sb ? b - sb : b + row_bytes - sb;
        out[b] = in[src];
    }
}

cudaError_t launch_destagger(size_t elem_size, size_t k, const void* img, const uint16_t* shift_host,
                             size_t h, size_t w, void* out, int device, cudaStream_t st) {
    (void)device;
    if (h == 0 || w == 0) return cudaSuccess;
    const size_t px_bytes = elem_size * k;
    const size_t row_bytes = px_bytes * w;
    if (h > 65535) return cudaErrorInvalidValue;
    if (h > static_cast<size_t>(kMaxRows)) {
        unsigned short* dsh = nullptr;
        cudaError_t e = cudaMallocAsync(&dsh, h * sizeof(unsigned short), st);
        if (e != cudaSuccess) return e;
        e = cudaMemcpyAsync(dsh, shift_host, h * sizeof(unsigned short), cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return e;
        dim3 grid(static_cast<unsigned>(std::min<size_t>((row_bytes + 255) / 256, 64)),
                  static_cast<unsigned>(h));
        launch(OB_FAM_DESTAGGER, destagger_bytes_dev_kernel, grid, 256, 0, st, static_cast<const uint8_t*>(img),
               static_cast<uint8_t*>(out), row_bytes, static_cast<unsigned>(px_bytes), dsh);
        e = cudaGetLastError();
        cudaFreeAsync(dsh, st);
        return e;
    }
    DestaggerParams p;
    p.in = static_cast<const uint8_t*>(img);
    p.out = static_cast<uint8_t*>(out);
    p.row_bytes = row_bytes;
    p.px_bytes = static_cast<unsigned>(px_bytes);
    p.H = static_cast<int>(h);
    for (int i = 0; i < kMaxRows; ++i) p.shift[i] = i < static_cast<int>(h) ? shift_host[i] : 0;
    const bool words = (row_bytes % 4 == 0) && ((reinterpret_cast<uintptr_t>(img) & 3u) == 0) &&
                       ((reinterpret_cast<uintptr_t>(out) & 3u) == 0) && row_bytes < (1ull << 31);
    if (words) {
        const size_t row_words = row_bytes / 4;
        dim3 grid(static_cast<unsigned>(std::min<size_t>((row_words + 255) / 256, 64)),
                  static_cast<unsigned>(h));
        launch(OB_FAM_DESTAGGER, destagger_words_kernel, grid, 256, 0, st, p);
    } else {
        dim3 grid(static_cast<unsigned>(std::min<size_t>((row_bytes + 255) / 256, 64)),
                  static_cast<unsigned>(h));
        launch(OB_FAM_DESTAGGER, destagger_bytes_kernel, grid, 256, 0, st, p);
    }
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// LUT construction on the device, in double.
// replaces impl::make_xyz_lut  ouster_core/src/xyzlut.cpp:11-89 (same operation order)
// ---------------------------------------------------------------------------------------------
struct LutParams {
    double b2l[16];
    double tr[16];
    double range_unit;
    unsigned long long w, h;
    int per_beam;
};

__global__ void make_lut_kernel(const __grid_constant__ LutParams p, const double* az_deg,
                                const double* alt_deg, double* dir, double* off) {
    const double kPi = 3.14159265358979323846;
    const unsigned long long n = p.w * p.h;
    const double b03 = p.b2l[3], b23 = p.b2l[11];
    double dist = b03;
    if (b23 != 0) dist = sqrt(__dadd_rn(__dmul_rn(b03, b03), __dmul_rn(b23, b23)));
    const double azimuth_radians = kPi * 2.0 / static_cast<double>(p.w);
    for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
         i < n; i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long row = i / p.w, col = i - row * p.w;
        double enc, az, alt;
        if (p.per_beam) {
            enc = __dsub_rn(2.0 * kPi, __dmul_rn(static_cast<double>(col), azimuth_radians));
            az = __ddiv_rn(__dmul_rn(-az_deg[row], kPi), 180.0);
            alt = __ddiv_rn(__dmul_rn(alt_deg[row], kPi), 180.0);
        } else {
            enc = 0;
            az = __ddiv_rn(__dmul_rn(az_deg[i], kPi), 180.0);
            alt = __ddiv_rn(__dmul_rn(alt_deg[i], kPi), 180.0);
        }
        const double ea = __dadd_rn(enc, az);
        double d[3], o[3];
        const double ca = cos(alt);
        d[0] = __dmul_rn(cos(ea), ca);
        d[1] = __dmul_rn(sin(ea), ca);
        d[2] = sin(alt);
        o[0] = __dsub_rn(__dmul_rn(cos(enc), b03), __dmul_rn(d[0], dist));
        o[1] = __dsub_rn(__dmul_rn(sin(enc), b03), __dmul_rn(d[1], dist));
        o[2] = __dadd_rn(__dmul_rn(-d[2], dist), b23);
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            double dj = __dadd_rn(__dadd_rn(__dmul_rn(d[0], p.tr[j * 4 + 0]),
                                            __dmul_rn(d[1], p.tr[j * 4 + 1])),
                                  __dmul_rn(d[2], p.tr[j * 4 + 2]));
            double oj = __dadd_rn(__dadd_rn(__dmul_rn(o[0], p.tr[j * 4 + 0]),
                                            __dmul_rn(o[1], p.tr[j * 4 + 1])),
                                  __dmul_rn(o[2], p.tr[j * 4 + 2]));
            oj = __dadd_rn(oj, p.tr[j * 4 + 3]);
            dir[i * 3 + j] = __dmul_rn(dj, p.range_unit);
            off[i * 3 + j] = __dmul_rn(oj, p.range_unit);
        }
    }
}

cudaError_t launch_make_lut(size_t w, size_t h, double range_unit, const double* b2l16,
                            const double* tr16, const double* az_dev, size_t n_az,
                            const double* alt_dev, size_t n_alt, double* dir_dev, double* off_dev,
                            cudaStream_t st) {
    LutParams p;
    for (int i = 0; i < 16; ++i) {
        p.b2l[i] = b2l16[i];
        p.tr[i] = tr16[i];
    }
    p.range_unit = range_unit;
    p.w = w;
    p.h = h;
    p.per_beam = (n_az == h && n_alt == h) ? 1 : 0;
    const size_t n = w * h;
    const int blocks = static_cast<int>(std::min<size_t>((n + 255) / 256, 1184));
    launch(OB_FAM_LUT, make_lut_kernel, std::max(blocks, 1), 256, 0, st, p, az_dev, alt_dev, dir_dev, off_dev);
    return cudaGetLastError();
}

__global__ void cast_f64_f32_kernel(const double* __restrict__ src, float* __restrict__ dst,
                                    size_t n) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x)
        dst[i] = static_cast<float>(src[i]);  // round-to-nearest, as Eigen's cast<float>()
}

cudaError_t launch_cast_f64_f32(const double* src, float* dst, size_t n, cudaStream_t st) {
    const int blocks = static_cast<int>(std::min<size_t>((n + 255) / 256, 1184));
    launch(OB_FAM_LUT, cast_f64_f32_kernel, std::max(blocks, 1), 256, 0, st, src, dst, n);
    return cudaGetLastError();
}

}  // namespace ob
