// ob_decode.cu -- K2: fused lidar-packet field decode -> row-major LidarFrame fields, with the
// per-row destagger of the range image(s) and the XYZ LUT projection done in the same pass.
//
// What it replaces (reference paths relative to /root/reference):
//   FieldDecodeInfo::get<T>                      ouster_core/include/ouster/core/field_decode_info.h:41-54
//   PacketFormat::block_field / col_field        ouster_core/src/parsing.cpp:628-675
//   FrameBatcher::parse_by_block / parse_by_col  ouster_core/src/lidar_frame.cpp:1422-1528
//   zero_fields / zero_header_cols               ouster_core/src/lidar_frame.cpp:1274-1278, 1371-1418
//   + cartesianT / destagger of the decoded range (impl/cartesian.h:36-66, impl/lidar_frame_impl.h:733-760)
//
// The reference walks every packet once per field (10 passes for dual return) with a transposing
// scatter; here a tile of TC frame columns (the columns of P whole packets) is brought into shared
// memory once by TMA bulk copies (one cp.async.bulk per packet, mbarrier-tracked, S-deep ring),
// every pixel is decoded once for all fields from registers, and the outputs leave as row-major
// coalesced stores (lane = frame column).  The XYZ projection re-reads the range words from the staged
// packet bytes and runs on 16-byte LUT loads / XYZ stores (lane = 16-byte chunk of a row).
//
// This file holds decode_kernel, the round-1 kernel (3 CTAs per SM, LUT rows loaded with LDG inside the
// compute loop).  Since round 2 the default is the pipelined, warp-specialised decode_pipe_kernel
// (ob_decode_pipe.cu); decode_kernel stays as the path for the launches that one does not take (frame
// width not a multiple of the tile, columns per packet not a power of two, unaligned LUT / XYZ pointers,
// range fields wider than a 32-bit plan) and as the A/B reference of the parity tests.
//
// Column map: frame column j takes its pixels from packet column col_src[j] (slot*cpp + c), or is
// zero-filled when col_src[j] < 0.  With the identity map (complete in-order frame) whole packets
// are bulk-copied; irregular groups are gathered column by column by the threads.


#include "ob_decode_tile.cuh"

namespace ob {

template <typename T>
__global__ void __launch_bounds__(384, 3) decode_kernel(const __grid_constant__ DecodeParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const DecodeLayout& L = p.L;
    const int tid = threadIdx.x, nthreads = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nthreads >> 5;
    const int S = p.stages;

    // ---- shared memory carve-up ----
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);   // kMaxStages
    TileCtl* ctl = reinterpret_cast<TileCtl*>(smem + 64);  // kMaxStages entries
    size_t off = 64 + static_cast<size_t>(kMaxStages) * sizeof(TileCtl);
    off = (off + 127) & ~static_cast<size_t>(127);
    uint8_t* stage0 = smem + off;

    if (tid == 0) {
        for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
        fence_proxy_async();
    }
    __syncthreads();

    const unsigned first = blockIdx.x;
    const unsigned n_my = first < p.n_tiles ? (p.n_tiles - first + gridDim.x - 1) / gridDim.x : 0;
    uint64_t pol_stream = 0;
    if (tid == 0) pol_stream = policy_evict_first();

    auto tile_of = [&](unsigned k, unsigned& f, unsigned& j0, unsigned& tc) {
        const unsigned t = first + k * gridDim.x;
        f = t / p.tiles_per_frame;
        j0 = (t - f * p.tiles_per_frame) * p.TC;
        tc = min(p.TC, L.W - j0);
    };
    // byte offset (inside a stage) of pixel 0 of tile column t
    auto col_offset = [&](unsigned t) -> int {
        const unsigned g = p.cpp_shift >= 0 ? (t >> p.cpp_shift) : (t / L.cpp);
        return static_cast<int>(g * p.pkt_stride_s + L.packet_header_size + (t - g * L.cpp) * L.col_size +
                                L.col_header_size);
    };

    auto issue = [&](unsigned k) {  // producer: thread 0
        unsigned f, j0, tc;
        tile_of(k, f, j0, tc);
        const int s = k % S;
        const DecodeFrame& fr = p.frames[f];
        TileCtl& c = ctl[s];
        uint8_t* st = stage0 + static_cast<size_t>(s) * p.stage_bytes;
        const bool identity = (fr.flags & kFrameIdentityMap) != 0;
        const bool bulk_ok = (fr.flags & kFrameBulkPackets) != 0;
        const unsigned n_groups = (tc + L.cpp - 1) / L.cpp;
        // regular tile: identity map, whole packets present -> no per-column bookkeeping
        if (identity && bulk_ok && (tc % L.cpp) == 0 && (j0 + tc) / L.cpp <= fr.n_slots) {
            c.regular = 1;
            mbar_expect_tx(&full[s], n_groups * L.packet_size);
            const unsigned slot0 = j0 / L.cpp;
            for (unsigned g = 0; g < n_groups; ++g)
                bulk_g2s_hint(st + static_cast<size_t>(g) * p.pkt_stride_s,
                              fr.packets + static_cast<size_t>(slot0 + g) * fr.packet_stride,
                              L.packet_size, &full[s], pol_stream);
            return;
        }
        c.regular = 0;
        uint32_t tx = 0;
        for (unsigned g = 0; g < n_groups; ++g) {
            const unsigned jg = j0 + g * L.cpp;
            const unsigned ncol = min(L.cpp, L.W - jg);
            bool fast = bulk_ok && ncol == L.cpp;
            int slot = -1;
            for (unsigned i = 0; i < ncol; ++i) {
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
            if (fast) tx += L.packet_size;
        }
        mbar_expect_tx(&full[s], tx);
        for (unsigned g = 0; g < n_groups; ++g) {
            if (!c.group_fast[g]) continue;
            const int slot = c.col_src[g * L.cpp] / static_cast<int>(L.cpp);
            bulk_g2s_hint(st + static_cast<size_t>(g) * p.pkt_stride_s,
                          fr.packets + static_cast<size_t>(slot) * fr.packet_stride, L.packet_size,
                          &full[s], pol_stream);
        }
    };

    // Warm L2 with the packets of a later tile (regular tiles only): with one stage per CTA the TMA
    // of tile k+S is issued only after tile k is consumed; having the bytes in L2 by then takes the
    // DRAM latency out of the mbarrier wait.
    auto prefetch_tile = [&](unsigned k, bool keep) {
        unsigned f, j0, tc;
        tile_of(k, f, j0, tc);
        const DecodeFrame& fr = p.frames[f];
        constexpr uint32_t regular = kFrameIdentityMap | kFrameBulkPackets;
        if ((fr.flags & regular) != regular || (tc % L.cpp) != 0 || (j0 + tc) / L.cpp > fr.n_slots) return;
        const unsigned slot0 = j0 / L.cpp, n_groups = tc / L.cpp;
        const uint64_t pol = keep ? policy_evict_last() : 0;
        for (unsigned g = 0; g < n_groups; ++g) {
            const uint8_t* src = fr.packets + static_cast<size_t>(slot0 + g) * fr.packet_stride;
            if (keep) bulk_prefetch_l2_hint(src, L.packet_size, pol);
            else bulk_prefetch_l2(src, L.packet_size);
        }
    };

    if (tid == 0) {
        const unsigned pre = min(n_my, static_cast<unsigned>(S));
        for (unsigned k = 0; k < pre; ++k) issue(k);
    }

    const bool aligned = p.word_aligned != 0;
    const unsigned n_ret = p.n_returns;
    const unsigned cds = L.channel_data_size;

    for (unsigned k = 0; k < n_my; ++k) {
        const int s = k % S;
        unsigned f, j0, tc;
        tile_of(k, f, j0, tc);
        const DecodeFrame& fr = p.frames[f];
        TileCtl& c = ctl[s];
        uint8_t* st = stage0 + static_cast<size_t>(s) * p.stage_bytes;

        mbar_wait(&full[s], (k / S) & 1);
        const bool regular = c.regular != 0;
        if (p.prefetch == 1 && tid == 32 && (k + S) < n_my) prefetch_tile(k + S, true);

        // ---- irregular groups: gather the columns with ordinary loads ----
        if (!regular) {
            const unsigned n_groups = (tc + L.cpp - 1) / L.cpp;
            bool any_slow = false;
            for (unsigned g = 0; g < n_groups; ++g) any_slow |= (c.group_fast[g] == 0);
            if (any_slow) {
                for (unsigned t = warp; t < tc; t += nwarps) {
                    const unsigned g = t / L.cpp;
                    if (c.group_fast[g]) continue;
                    const int src = c.col_src[t];
                    if (src < 0) continue;
                    const int sl = src / static_cast<int>(L.cpp), ci = src - sl * static_cast<int>(L.cpp);
                    const uint8_t* gsrc = fr.packets + static_cast<size_t>(sl) * fr.packet_stride +
                                          L.packet_header_size + static_cast<size_t>(ci) * L.col_size;
                    uint8_t* dst = st + static_cast<size_t>(g) * p.pkt_stride_s + L.packet_header_size +
                                   static_cast<size_t>(t - g * L.cpp) * L.col_size;
                    // the column plus the 8 bytes a trailing field read may touch (clamped to the packet)
                    const size_t col_end = L.packet_header_size + static_cast<size_t>(ci + 1) * L.col_size;
                    const size_t extra = min(static_cast<size_t>(8), L.packet_size - col_end);
                    const unsigned nbytes = L.col_size + static_cast<unsigned>(extra);
                    if (aligned && ((reinterpret_cast<uintptr_t>(gsrc) & 3u) == 0)) {
                        for (unsigned b = lane * 4; b + 4 <= nbytes; b += 128)
                            *reinterpret_cast<uint32_t*>(dst + b) = *reinterpret_cast<const uint32_t*>(gsrc + b);
                        for (unsigned b = (nbytes & ~3u) + lane; b < nbytes; b += 32) dst[b] = gsrc[b];
                    } else {
                        for (unsigned b = lane; b < nbytes; b += 32) dst[b] = gsrc[b];
                    }
                }
                __syncthreads();
            }
        }

        // ---- column headers (timestamp / measurement_id / status) ----
        if (fr.timestamp != nullptr || fr.measurement_id != nullptr || fr.status != nullptr) {
            for (unsigned t = tid; t < tc; t += nthreads) {
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

        // ---- phase A: decode; lane = frame column, warp = row (strided), fields outermost ----
        // narrow tiles (fewer than 32 columns) with a compile-time layout: a warp covers RW rows
        // per instruction (lane = column + tc * sub-row) instead of leaving lanes idle
        const unsigned RW = (p.layout_id != 0 && tc < 32u && (32u % tc) == 0u) ? 32u / tc : 1u;
        for (unsigned cg = 0; cg * 32 < tc; ++cg) {
            const unsigned t = RW > 1 ? (static_cast<unsigned>(lane) % tc) : cg * 32 + lane;
            const unsigned sub = RW > 1 ? static_cast<unsigned>(lane) / tc : 0u;
            const bool lane_on = t < tc;
            const unsigned tt = lane_on ? t : 0;
            const int co = regular ? col_offset(tt) : c.col_off[tt];
            const bool col_valid = co >= 0;
            const uint8_t* px0 = st + (col_valid ? co : col_offset(tt));
            const size_t pix0 = static_cast<size_t>(j0) + tt;
            if (p.layout_id != 0) {
                uint8_t* outp[kMaxSlots];
#pragma unroll
                for (int i = 0; i < kMaxSlots; ++i)
                    outp[i] = p.slot_field[i] >= 0 ? static_cast<uint8_t*>(fr.fields[p.slot_field[i]]) : nullptr;
                uint32_t* rdp2[2] = {fr.rd[0], fr.rd[1]};
                const bool full = regular && (RW > 1 || (cg + 1) * 32u <= tc);
                const unsigned col = static_cast<unsigned>(pix0);
                const unsigned row0 = static_cast<unsigned>(warp) * RW + sub, rstep = static_cast<unsigned>(nwarps) * RW;
                const int all = static_output_mode(p, fr);
                switch (p.layout_id) {
                    case 1: decode_static_tile<1>(full, all, px0, col_valid, lane_on, outp, rdp2, col, L.W, L.H, row0, rstep, p); break;
                    case 2: decode_static_tile<2>(full, all, px0, col_valid, lane_on, outp, rdp2, col, L.W, L.H, row0, rstep, p); break;
                    case 3: decode_static_tile<3>(full, all, px0, col_valid, lane_on, outp, rdp2, col, L.W, L.H, row0, rstep, p); break;
                    case 4: decode_static_tile<4>(full, all, px0, col_valid, lane_on, outp, rdp2, col, L.W, L.H, row0, rstep, p); break;
                    default: decode_static_tile<5>(full, all, px0, col_valid, lane_on, outp, rdp2, col, L.W, L.H, row0, rstep, p); break;
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
                if (pl.fast && es <= 4) {
                    const uint32_t zv = (fd.zero_pattern & 0xffffu) | ((fd.zero_pattern & 0xffffu) << 16);
                    const bool ho = out != nullptr, hr = rdp != nullptr;
                    const bool full = regular && (cg + 1) * 32u <= tc;
                    if (full) {
                        if (es == 4) decode_rows_dispatch<4, true>(ho, hr, px0, cds, pl, true, zv, true, out, pix0, L.W, L.H, warp, nwarps, rdp, p);
                        else if (es == 2) decode_rows_dispatch<2, true>(ho, hr, px0, cds, pl, true, zv, true, out, pix0, L.W, L.H, warp, nwarps, rdp, p);
                        else decode_rows_dispatch<1, true>(ho, hr, px0, cds, pl, true, zv, true, out, pix0, L.W, L.H, warp, nwarps, rdp, p);
                    } else {
                        if (es == 4) decode_rows_dispatch<4, false>(ho, hr, px0, cds, pl, col_valid, zv, lane_on, out, pix0, L.W, L.H, warp, nwarps, rdp, p);
                        else if (es == 2) decode_rows_dispatch<2, false>(ho, hr, px0, cds, pl, col_valid, zv, lane_on, out, pix0, L.W, L.H, warp, nwarps, rdp, p);
                        else decode_rows_dispatch<1, false>(ho, hr, px0, cds, pl, col_valid, zv, lane_on, out, pix0, L.W, L.H, warp, nwarps, rdp, p);
                    }
                } else {  // wide or unaligned fields: generic 64-bit extraction
                    for (unsigned row = warp; row < L.H; row += nwarps) {
                        if (!lane_on) continue;
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

        if (p.prefetch == 2 && tid == 32 && (k + S) < n_my) prefetch_tile(k + S, false);

        // ---- phase B: XYZ; lane = 16-byte chunk of a row segment, ranges re-read from the stage ----
        const void* lut_dir_f = fr.lut_dir != nullptr ? fr.lut_dir : p.lut_dir;
        const void* lut_off_f = fr.lut_dir != nullptr ? fr.lut_off : p.lut_off;
        if (lut_dir_f != nullptr && n_ret > 0) {
            const T* dir = static_cast<const T*>(lut_dir_f);
            const T* offs = static_cast<const T*>(lut_off_f);
            constexpr int VN = 16 / sizeof(T);  // scalars per 16-byte chunk
            const DecodeParams::Plan& pl0 = p.plan[p.range_field[0]];
            const DecodeParams::Plan& pl1 = p.plan[p.range_field[n_ret > 1 ? 1 : 0]];
            T* xo0 = static_cast<T*>(fr.xyz[0]);
            T* xo1 = n_ret > 1 ? static_cast<T*>(fr.xyz[1]) : nullptr;
            if (p.vec_ok && (tc % 4u) == 0 && p.plan_ranges_fast) {
                const unsigned nvr = 3u * tc / VN;  // 16-byte chunks per row segment
                // every thread owns one chunk position q of the row segment and walks down the rows:
                // pixel indices, column offsets, masks and element->pixel selects are loop invariants
                const unsigned rows_per_pass = static_cast<unsigned>(nthreads) / nvr;
                if (rows_per_pass > 0 && static_cast<unsigned>(tid) < rows_per_pass * nvr) {
                    const unsigned row0 = static_cast<unsigned>(tid) / nvr;
                    const unsigned q = static_cast<unsigned>(tid) - row0 * nvr;
                    const unsigned e0 = q * VN;
                    const unsigned p0 = e0 / 3u;       // first pixel touched by this chunk
                    const unsigned k0 = e0 - 3u * p0;  // component of element 0 inside pixel p0
                    const unsigned p1 = (p0 + 1 < tc) ? p0 + 1 : p0;
                    const int co0 = regular ? col_offset(p0) : c.col_off[p0];
                    const int co1 = regular ? col_offset(p1) : c.col_off[p1];
                    const bool v0 = co0 >= 0, v1 = co1 >= 0;
                    const uint32_t* wa0 = reinterpret_cast<const uint32_t*>(st + (v0 ? co0 : 0) + static_cast<size_t>(row0) * cds);
                    const uint32_t* wb0 = reinterpret_cast<const uint32_t*>(st + (v1 ? co1 : 0) + static_cast<size_t>(row0) * cds);
                    const unsigned wstep = rows_per_pass * cds / 4u;
                    const size_t ebase = (static_cast<size_t>(row0) * L.W + j0) * 3 + static_cast<size_t>(q) * VN;
                    const size_t estep = static_cast<size_t>(rows_per_pass) * L.W * 3;
                    const bool simple = (pl0.mb | pl1.mb | pl0.rs | pl1.rs) == 0 && pl0.d == 0 && pl1.d == 0;
                    const bool both = xo0 != nullptr && xo1 != nullptr;
                    if (simple && v0 && v1 && both)
                        project_rows<T, true, true>(dir + ebase, offs + ebase, xo0 + ebase, xo1 + ebase, estep,
                                                    wa0, wb0, wstep, pl0, pl1, true, true, k0, row0, rows_per_pass, L.H);
                    else
                        project_rows<T, false, false>(dir + ebase, offs + ebase, xo0 ? xo0 + ebase : nullptr,
                                                      xo1 ? xo1 + ebase : nullptr, estep, wa0, wb0, wstep, pl0, pl1,
                                                      v0, v1, k0, row0, rows_per_pass, L.H);
                }
            } else {
                for (unsigned idx = tid; idx < L.H * tc; idx += nthreads) {
                    const unsigned row = idx / tc, t = idx - row * tc;
                    const int co = regular ? col_offset(t) : c.col_off[t];
                    const size_t ebase = (static_cast<size_t>(row) * L.W + j0 + t) * 3;
                    for (unsigned r = 0; r < n_ret; ++r) {
                        T* xo = static_cast<T*>(fr.xyz[r]);
                        if (xo == nullptr) continue;
                        const DecodeField& fd = L.fields[p.range_field[r]];
                        const uint32_t rv = co < 0 ? 0u
                                                   : static_cast<uint32_t>(extract_smem(st + co + row * cds, fd, aligned));
#pragma unroll
                        for (int cidx = 0; cidx < 3; ++cidx)
                            xo[ebase + cidx] = project1(rv, dir[ebase + cidx], offs[ebase + cidx]);
                    }
                }
            }
        }
        __syncthreads();  // every warp is done with this stage
        if (tid == 0 && (k + S) < n_my) issue(k + S);
    }
}

// Fills the launch parameters shared by both K2 kernels.  `pipe`: tile geometry of the pipelined kernel
// (ob_decode_pipe.cu): at most 64 columns per tile so that a LUT row segment fits one TMA box.
cudaError_t make_decode_params(const DecodeLaunch& a, int device, bool pipe, DecodeParams& p) {
    const Tunables& tn = tunables(device);
    const DecodeLayout& L = *a.layout_host;
    if (L.cpp == 0 || L.H == 0 || L.W == 0 || L.cpp > static_cast<uint32_t>(kMaxTileCols))
        return cudaErrorInvalidValue;
    p.L = L;
    p.frames = a.frames_dev;
    p.lut_dir = a.lut_dir;
    p.lut_off = a.lut_off;
    p.n_frames = a.n_frames;
    // bytes reserved per packet in a stage.  decode_kernel: + 16 slack for trailing 8-byte field reads; the
    // pipelined kernel packs the packets back to back (an over-read lands in the next packet's header, masked
    // off anyway) and keeps one 16-byte slack after the last stage -- that is what lets a 4-slot LUT ring fit
    p.pkt_stride_s = pipe ? ((L.packet_size + 15) & ~15u) : ((L.packet_size + 16 + 15) & ~15u);
    if (pipe) {
        uint32_t ncw, ctas;
        decode_pipe_shape(L, device, &p.P, &ncw, &ctas);
    } else if (tn.decode_tile_packets > 0) {
        p.P = static_cast<uint32_t>(tn.decode_tile_packets);
    } else {
        // auto: as many packets as fit a ~68 KB stage (3 CTAs per SM), power of two, at least 32 columns
        p.P = 1;
        while (p.P * 2 * p.pkt_stride_s <= 68u * 1024u && p.P * 2 * L.cpp <= static_cast<uint32_t>(kMaxTileCols)) p.P *= 2;
    }
    p.P = std::max<uint32_t>(1, std::min<uint32_t>(p.P, static_cast<uint32_t>(kMaxTileCols) / L.cpp));
    p.TC = p.P * L.cpp;
    p.tiles_per_frame = (L.W + p.TC - 1) / p.TC;
    p.n_tiles = p.tiles_per_frame * a.n_frames;
    p.stage_bytes = (p.P * p.pkt_stride_s + 127) & ~127u;
    p.stages = std::min(std::max(tn.decode_stages, 1), kMaxStages);
    const bool word_aligned = (L.packet_header_size % 4 == 0) && (L.col_header_size % 4 == 0) &&
                              (L.channel_data_size % 4 == 0) && (L.col_size % 4 == 0);
    p.word_aligned = word_aligned ? 1 : 0;
    p.n_returns = 0;
    for (uint32_t i = 0; i < L.n_fields; ++i) {
        if (L.fields[i].range_return >= 0)
            p.n_returns = std::max<uint32_t>(p.n_returns, L.fields[i].range_return + 1);
    }
    // per-field 32-bit extraction plans: core = ((window & mask) >> tz), value = core << (tz - shift)
    for (uint32_t i = 0; i < OB_MAX_FIELDS; ++i) {
        DecodeParams::Plan pl{};
        if (i < L.n_fields && word_aligned) {
            const DecodeField& f = L.fields[i];
            const uint64_t mask = f.mask;
            if (mask == 0) {
                pl.fast = 1;  // always zero
            } else {
                const int tz = __builtin_ctzll(mask);
                const uint64_t core = mask >> tz;
                if (core <= 0xffffffffull) {
                    const uint32_t a = (f.offset & 3u) * 8u + static_cast<uint32_t>(tz);  // bit index from word f.offset/4
                    pl.wa = (f.offset >> 2) + a / 32u;
                    pl.rs = a % 32u;
                    const unsigned __int128 m96 = static_cast<unsigned __int128>(core) << pl.rs;
                    pl.ma = static_cast<uint32_t>(m96 & 0xffffffffu);
                    pl.mb = static_cast<uint32_t>((m96 >> 32) & 0xffffffffu);
                    const int d = tz - f.shift;
                    pl.d = d > 31 ? 32 : (d < -31 ? -32 : d);
                    pl.fast = (d > 31 || d < -31) ? 0 : 1;
                }
            }
        }
        p.plan[i] = pl;
    }
    // ---- compile-time layout match: every runtime field must land on a distinct slot ----
    p.layout_id = 0;
    p.layout_all = 0;
    for (int i = 0; i < kMaxSlots; ++i) p.slot_field[i] = -1;
    if (word_aligned && !tn.decode_runtime_plans && static_cast<uint64_t>(L.H) * L.W < (1ull << 30)) {
        auto try_layout = [&](int id, const PxSlot* slots, int n_slots, uint32_t cds) {
            if (p.layout_id != 0 || L.channel_data_size != cds || L.n_fields == 0) return;
            signed char map[kMaxSlots];
            for (int i = 0; i < kMaxSlots; ++i) map[i] = -1;
            for (uint32_t i = 0; i < L.n_fields; ++i) {
                const DecodeField& f = L.fields[i];
                if (f.mask == 0 || f.zero_pattern != 0) return;
                const int tz = __builtin_ctzll(f.mask);
                const uint64_t core = f.mask >> tz;
                if ((core & (core + 1)) != 0) return;  // not a contiguous bit field
                const int bits = __builtin_popcountll(core);
                const int up = tz - f.shift;
                const uint32_t lsb = f.offset * 8u + static_cast<uint32_t>(tz);
                int hit = -1;
                for (int j = 0; j < n_slots; ++j) {
                    const PxSlot& sl = slots[j];
                    if (sl.bits != 0 && sl.lsb == lsb && sl.bits == bits && sl.up == up && sl.es == f.elem_size &&
                        sl.ret == f.range_return && map[j] < 0) {
                        hit = j;
                        break;
                    }
                }
                if (hit < 0) return;
                map[hit] = static_cast<signed char>(i);
            }
            p.layout_id = static_cast<uint32_t>(id);
            p.layout_all = 1;
            for (int i = 0; i < kMaxSlots; ++i) p.slot_field[i] = map[i];
            for (int j = 0; j < n_slots; ++j) p.layout_all &= map[j] >= 0 ? 1u : 0u;
        };
        try_layout(1, PxLayout<1>::s, PxLayout<1>::n, PxLayout<1>::cds);
        try_layout(2, PxLayout<2>::s, PxLayout<2>::n, PxLayout<2>::cds);
        try_layout(3, PxLayout<3>::s, PxLayout<3>::n, PxLayout<3>::cds);
        try_layout(4, PxLayout<4>::s, PxLayout<4>::n, PxLayout<4>::cds);
        try_layout(5, PxLayout<5>::s, PxLayout<5>::n, PxLayout<5>::cds);
    }
    p.cpp_shift = -1;
    for (int b = 0; b < 8; ++b)
        if ((1u << b) == L.cpp) p.cpp_shift = b;
    p.range_field[0] = p.range_field[1] = 0;
    p.plan_ranges_fast = 1;
    for (uint32_t i = 0; i < L.n_fields; ++i) {
        const int r = L.fields[i].range_return;
        if (r >= 0 && r < OB_MAX_RETURNS) {
            p.range_field[r] = i;
            if (!p.plan[i].fast) p.plan_ranges_fast = 0;
        }
    }
    p.prefetch = static_cast<uint32_t>(std::max(0, tn.decode_prefetch));
    p.vec_ok = (L.W % 4 == 0) ? 1 : 0;  // the C-ABI glue (DecodeLaunch::vec_ok) also checks pointer alignment
    p.has_shift = a.shift_host != nullptr ? 1 : 0;
    for (int i = 0; i < kMaxRows; ++i)
        p.shift[i] = (a.shift_host != nullptr && i < static_cast<int>(L.H)) ? a.shift_host[i] : 0;
    if (a.shift_host != nullptr && L.H > static_cast<uint32_t>(kMaxRows)) return cudaErrorInvalidValue;
    if (!a.vec_ok) p.vec_ok = 0;

    return cudaSuccess;
}

cudaError_t launch_decode(const DecodeLaunch& a, int device, cudaStream_t st) {
    const Tunables& tn = tunables(device);
    const DecodeLayout& L = *a.layout_host;
    DecodeParams p;
    if (tn.decode_pipe) {
        cudaError_t e = make_decode_params(a, device, true, p);
        if (e != cudaSuccess) return e;
        if (decode_pipe_eligible(p, a, device)) return launch_decode_pipe(p, a, device, st);
    }
    cudaError_t e0 = make_decode_params(a, device, false, p);
    if (e0 != cudaSuccess) return e0;
    const size_t rtile_bytes = 0;  // ranges are re-read from the staged packets in phase B
    size_t ctl_off = 64 + static_cast<size_t>(kMaxStages) * sizeof(TileCtl);
    ctl_off = (ctl_off + 127) & ~static_cast<size_t>(127);
    size_t smem = ctl_off + static_cast<size_t>(p.stages) * p.stage_bytes + rtile_bytes;
    while (smem > 227 * 1024 && p.stages > 1) {
        p.stages--;
        smem = ctl_off + static_cast<size_t>(p.stages) * p.stage_bytes + rtile_bytes;
    }
    if (smem > 227 * 1024) return cudaErrorInvalidValue;
    int threads = tn.decode_threads;
    const int grid = static_cast<int>(
        std::min<uint32_t>(p.n_tiles, static_cast<uint32_t>(tn.sm_count) * tn.decode_ctas_per_sm));
    auto kern = a.lut_dtype == OB_F64 ? decode_kernel<double> : decode_kernel<float>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    launch(OB_FAM_DECODE, kern, std::max(grid, 1), threads, smem, st, p);
    return cudaGetLastError();
}

}  // namespace ob
