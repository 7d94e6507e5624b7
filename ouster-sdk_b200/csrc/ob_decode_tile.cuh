// ob_decode_tile.cuh -- device code shared by the K2 kernels (ob_decode.cu, ob_decode_pipe.cu):
// launch parameters, per-stage tile bookkeeping, the per-field extraction plans, the compile-time
// pixel layouts and the phase-A row loops.  See ob_decode.cu for what the kernels replace.
#pragma once
#include <algorithm>
#include <type_traits>
#include <utility>

#include "ob_internal.h"
#include "ob_ptx.cuh"

namespace ob {

constexpr int kMaxTileCols = 128;
constexpr int kMaxStages = 4;

struct DecodeParams {
    DecodeLayout L;
    const DecodeFrame* frames;
    const void* lut_dir;
    const void* lut_off;
    uint32_t n_frames, tiles_per_frame, n_tiles;
    uint32_t TC, P;             // tile columns (= P * cpp), packets per tile
    uint32_t pkt_stride_s;      // bytes reserved per packet in a stage (multiple of 16)
    uint32_t stage_bytes, stages;
    uint32_t word_aligned;      // wire layout is 4-byte aligned everywhere
    uint32_t n_returns;         // returns with a range field tagged
    uint32_t vec_ok;            // XYZ rows are 16-byte aligned (W % 4 == 0, aligned pointers)
    uint32_t has_shift;
    int32_t cpp_shift;          // log2(columns_per_packet) or -1
    uint32_t range_field[OB_MAX_RETURNS];  // index of the range field of each return
    uint32_t plan_ranges_fast;  // the range fields have 32-bit plans
    uint32_t prefetch;          // L2 prefetch of the next tile (Tunables::decode_prefetch)
    uint32_t layout_id;         // > 0: compile-time pixel layout (see PxLayout); 0: runtime plans
    signed char slot_field[16]; // layout slot -> index into fields[] (or -1: field not in the frame)
    uint32_t layout_all;        // every slot of the layout is a decoder field
    struct Plan {        // per-field extraction plan, precomputed on the host (see make_plan)
        uint32_t wa;     // aligned 32-bit word (from the pixel start) holding the field's LSB
        uint32_t ma, mb; // masks of that word and the next one
        uint32_t rs;     // funnel right shift (0..31) that brings the field's LSB to bit 0
        int32_t d;       // post shift: >= 0 left, < 0 right (upshift / partial down-shift)
        uint32_t fast;   // 1: 32-bit plan valid (value fits 32 bits, layout word aligned)
    } plan[OB_MAX_FIELDS];
    unsigned short shift[kMaxRows];
};

struct TileCtl {  // per-stage bookkeeping written by the producer thread
    int regular;                // 1: identity map, whole packets present (tables below unused)
    int col_src[kMaxTileCols];  // source packet column (slot*cpp + c) or -1
    int col_off[kMaxTileCols];  // byte offset of the column's pixel 0 inside the stage, or -1
    unsigned char group_fast[kMaxTileCols];
};

// FieldDecodeInfo::get: 8-byte little-endian load at `offset`, mask, shift (caller truncates)
__device__ __forceinline__ uint64_t apply_mask_shift(uint32_t lo, uint32_t hi, const DecodeField& f) {
    uint64_t word = (static_cast<uint64_t>(hi) << 32) | lo;
    word &= f.mask;
    if (f.shift > 0) word >>= f.shift;
    else if (f.shift < 0) word <<= -f.shift;
    return word;
}

__device__ __forceinline__ uint64_t extract_smem(const uint8_t* px, const DecodeField& f, bool aligned) {
    const uint8_t* p = px + f.offset;
    if (aligned && (f.offset & 3u) == 0)
        return apply_mask_shift(*reinterpret_cast<const uint32_t*>(p),
                                *reinterpret_cast<const uint32_t*>(p + 4), f);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        lo |= static_cast<uint32_t>(p[i]) << (8 * i);
        hi |= static_cast<uint32_t>(p[4 + i]) << (8 * i);
    }
    return apply_mask_shift(lo, hi, f);
}

__device__ __forceinline__ void store_elem(void* base, size_t idx, uint32_t es, uint64_t v) {
    switch (es) {
        case 1: static_cast<uint8_t*>(base)[idx] = static_cast<uint8_t>(v); break;
        case 2: static_cast<uint16_t*>(base)[idx] = static_cast<uint16_t>(v); break;
        case 4: static_cast<uint32_t*>(base)[idx] = static_cast<uint32_t>(v); break;
        case 8: static_cast<uint64_t*>(base)[idx] = v; break;
        default: {  // 6 bytes: 3 x 16 bit (float3x16_t, RGB)
            uint16_t* q = static_cast<uint16_t*>(base) + idx * 3;
            q[0] = static_cast<uint16_t>(v);
            q[1] = static_cast<uint16_t>(v >> 16);
            q[2] = static_cast<uint16_t>(v >> 32);
        }
    }
}

__device__ __forceinline__ uint64_t zero_value(const DecodeField& f) {
    const uint64_t z = f.zero_pattern & 0xffffu;
    return z | (z << 16) | (z << 32) | (z << 48);
}

__device__ __forceinline__ float project1(uint32_t r, float d, float o) {
    return r == 0 ? 0.0f : __fadd_rn(__fmul_rn(static_cast<float>(r), d), o);
}
__device__ __forceinline__ double project1(uint32_t r, double d, double o) {
    return r == 0 ? 0.0 : __dadd_rn(__dmul_rn(static_cast<double>(r), d), o);
}
// range already converted: r * dir + ofs with the reference's two roundings (the caller handles r == 0)
__device__ __forceinline__ float project_nz(float r, float d, float o) { return __fadd_rn(__fmul_rn(r, d), o); }
__device__ __forceinline__ double project_nz(double r, double d, double o) { return __dadd_rn(__dmul_rn(r, d), o); }

// Row loop of phase A for one field.  Compile-time specialisations remove every per-pixel branch:
//   ES      destination element size (1, 2, 4)
//   NEED_B  the field straddles two aligned 32-bit words
//   SHIFTED the value needs the extra up/down shift (low-bandwidth profiles, custom tables)
//   MODE    1 = plain image only, 2 = plain + destaggered range, 3 = destaggered range only
//   FULL    every lane holds a present column (complete tile): no predication, no zero fill
// The main loop handles 4 rows per trip with a single bounds test; all addresses advance by
// loop-invariant strides.  ~9 instructions per pixel in the common case.
template <int ES, bool NEED_B, bool SHIFTED, int MODE, bool FULL>
__device__ __forceinline__ void decode_rows(const uint8_t* px0, unsigned cds, const DecodeParams::Plan& pl,
                                            bool col_valid, uint32_t zv, bool lane_on, uint8_t* out,
                                            size_t pix0, unsigned W, unsigned H, int warp, int nwarps,
                                            uint32_t* rdp, const DecodeParams& p) {
    constexpr bool HAS_OUT = MODE != 3, RR = MODE != 1;
    // output pointers come from the frame table (generic): tell the compiler they are global memory
    if (HAS_OUT) __builtin_assume(__isGlobal(out));
    if (RR) __builtin_assume(__isGlobal(rdp));
    const uint32_t lsh = pl.d > 0 ? static_cast<uint32_t>(pl.d) : 0u;
    const uint32_t rsh = pl.d < 0 ? static_cast<uint32_t>(-pl.d) : 0u;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(px0 + static_cast<size_t>(warp) * cds) + pl.wa;
    const unsigned wstep = static_cast<unsigned>(nwarps) * cds / 4u;
    uint8_t* o = HAS_OUT ? out + (static_cast<size_t>(warp) * W + pix0) * ES : nullptr;
    const size_t ostep = static_cast<size_t>(nwarps) * W * ES;
    uint32_t* rrow = RR ? rdp + static_cast<size_t>(warp) * W : nullptr;
    const size_t rstep = static_cast<size_t>(nwarps) * W;
    const int col = static_cast<int>(pix0), Wi = static_cast<int>(W);
    const bool has_shift = p.has_shift != 0;

    auto body = [&](unsigned row) {
        const uint32_t a = w[0] & pl.ma;
        uint32_t v;
        if (NEED_B) v = __funnelshift_r(a, w[1] & pl.mb, pl.rs);
        else v = a >> pl.rs;
        if (SHIFTED) v = (v << lsh) >> rsh;
        if (!FULL) v = col_valid ? v : zv;
        if (FULL || lane_on) {
            if (HAS_OUT) {
                if (ES == 4) *reinterpret_cast<uint32_t*>(o) = v;
                else if (ES == 2) *reinterpret_cast<uint16_t*>(o) = static_cast<uint16_t>(v);
                else *o = static_cast<uint8_t>(v);
            }
            if (RR) {
                int dcol = col + (has_shift ? p.shift[row] : 0);
                dcol = dcol >= Wi ? dcol - Wi : dcol;
                rrow[dcol] = v;
            }
        }
        w += wstep;
        if (HAS_OUT) o += ostep;
        if (RR) rrow += rstep;
    };
    unsigned row = warp;
    const unsigned nw = static_cast<unsigned>(nwarps);
    for (; row + 3u * nw < H; row += 4u * nw) {
        body(row);
        body(row + nw);
        body(row + 2u * nw);
        body(row + 3u * nw);
    }
    for (; row < H; row += nw) body(row);
}

template <int ES, bool NEED_B, bool SHIFTED, bool FULL>
__device__ __forceinline__ void decode_rows_mode(bool has_out, bool has_rd, const uint8_t* px0, unsigned cds,
                                                 const DecodeParams::Plan& pl, bool col_valid, uint32_t zv,
                                                 bool lane_on, uint8_t* out, size_t pix0, unsigned W,
                                                 unsigned H, int warp, int nwarps, uint32_t* rdp,
                                                 const DecodeParams& p) {
    if (has_out && has_rd)
        decode_rows<ES, NEED_B, SHIFTED, 2, FULL>(px0, cds, pl, col_valid, zv, lane_on, out, pix0, W, H, warp, nwarps, rdp, p);
    else if (has_out)
        decode_rows<ES, NEED_B, SHIFTED, 1, FULL>(px0, cds, pl, col_valid, zv, lane_on, out, pix0, W, H, warp, nwarps, rdp, p);
    else if (has_rd)
        decode_rows<ES, NEED_B, SHIFTED, 3, FULL>(px0, cds, pl, col_valid, zv, lane_on, out, pix0, W, H, warp, nwarps, rdp, p);
}

template <int ES, bool FULL>
__device__ __forceinline__ void decode_rows_dispatch(bool has_out, bool has_rd, const uint8_t* px0,
                                                     unsigned cds, const DecodeParams::Plan& pl,
                                                     bool col_valid, uint32_t zv, bool lane_on,
                                                     uint8_t* out, size_t pix0, unsigned W, unsigned H,
                                                     int warp, int nwarps, uint32_t* rdp,
                                                     const DecodeParams& p) {
    const bool need_b = pl.mb != 0, shifted = pl.d != 0;
    if (need_b) {
        if (shifted) decode_rows_mode<ES, true, true, FULL>(has_out, has_rd, px0, cds, pl, col_valid, zv, lane_on, out, pix0, W, H, warp, nwarps, rdp, p);
        else decode_rows_mode<ES, true, false, FULL>(has_out, has_rd, px0, cds, pl, col_valid, zv, lane_on, out, pix0, W, H, warp, nwarps, rdp, p);
    } else {
        if (shifted) decode_rows_mode<ES, false, true, FULL>(has_out, has_rd, px0, cds, pl, col_valid, zv, lane_on, out, pix0, W, H, warp, nwarps, rdp, p);
        else decode_rows_mode<ES, false, false, FULL>(has_out, has_rd, px0, cds, pl, col_valid, zv, lane_on, out, pix0, W, H, warp, nwarps, rdp, p);
    }
}

// Phase B row walk of one thread: chunk position fixed, rows strided.  SIMPLE: both range fields
// are `word & mask` (no straddle, no shift); BOTH: both returns requested and both pixels present.
template <typename T, bool SIMPLE, bool BOTH>
__device__ __forceinline__ void project_rows(const T* dir, const T* offs, T* xo0, T* xo1, size_t estep,
                                             const uint32_t* wa, const uint32_t* wb, unsigned wstep,
                                             const DecodeParams::Plan& pl0, const DecodeParams::Plan& pl1,
                                             bool v0, bool v1, unsigned k0, unsigned row0,
                                             unsigned rows_per_pass, unsigned H) {
    using V = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
    constexpr int VN = 16 / sizeof(T);
    auto rng = [](const uint32_t* w, const DecodeParams::Plan& pl, bool valid) -> uint32_t {
        const uint32_t a = w[pl.wa] & pl.ma;
        if (SIMPLE) return a;
        const uint32_t b = pl.mb ? (w[pl.wa + 1] & pl.mb) : 0u;
        uint32_t v = __funnelshift_r(a, b, pl.rs);
        v = pl.d >= 0 ? (v << pl.d) : (v >> (-pl.d));
        return valid ? v : 0u;
    };
    // element e of the chunk belongs to the chunk's first pixel iff k0 + e < 3
    bool first[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) first[e] = (k0 + e) < 3u;
    __builtin_assume(__isGlobal(dir));
    __builtin_assume(__isGlobal(offs));
    if (BOTH || xo0 != nullptr) __builtin_assume(__isGlobal(xo0));
    if (BOTH || xo1 != nullptr) __builtin_assume(__isGlobal(xo1));
    // software pipeline: the LUT chunk of the next row is in flight while this row is computed
    V dv = *reinterpret_cast<const V*>(dir);
    V ov = *reinterpret_cast<const V*>(offs);
#pragma unroll 2
    for (unsigned row = row0; row < H; row += rows_per_pass) {
        V dvn = dv, ovn = ov;
        if (row + rows_per_pass < H) {
            dvn = *reinterpret_cast<const V*>(dir + estep);
            ovn = *reinterpret_cast<const V*>(offs + estep);
        }
        const T* de = reinterpret_cast<const T*>(&dv);
        const T* oe = reinterpret_cast<const T*>(&ov);
        if (BOTH || xo0 != nullptr) {
            const uint32_t ra = rng(wa, pl0, v0), rb = rng(wb, pl0, v1);
            V outv;
            T* o2 = reinterpret_cast<T*>(&outv);
#pragma unroll
            for (int e = 0; e < VN; ++e) o2[e] = project1(first[e] ? ra : rb, de[e], oe[e]);
            *reinterpret_cast<V*>(xo0) = outv;
            xo0 += estep;
        }
        if (BOTH || xo1 != nullptr) {
            const uint32_t ra = rng(wa, pl1, v0), rb = rng(wb, pl1, v1);
            V outv;
            T* o2 = reinterpret_cast<T*>(&outv);
#pragma unroll
            for (int e = 0; e < VN; ++e) o2[e] = project1(first[e] ? ra : rb, de[e], oe[e]);
            *reinterpret_cast<V*>(xo1) = outv;
            xo1 += estep;
        }
        wa += wstep;
        wb += wstep;
        dir += estep;
        offs += estep;
        dv = dvn;
        ov = ovn;
    }
}

// ---------------------------------------------------------------------------------------------
// Compile-time pixel layouts.  The channel-data block of the standard profiles is a fixed bit
// field (parsing.cpp:170-363); with the layout known at compile time a pixel is read once
// (cds/4 LDS) and every field is one or two ALU instructions and one store -- no per-field pass,
// no per-field branches.  A slot is (first bit, width, up-shift, destination element size, return
// whose range image it is or -1); names do not matter, so profiles that only rename a slot
// (NEAR_IR / ZONE_MASK) share a layout.  launch_decode() matches the decoder's runtime field
// table against these slots; anything else (custom profiles, RAW32_WORDn, RGB, wider
// destinations) keeps the runtime-plan path above.
// ---------------------------------------------------------------------------------------------
struct PxSlot {
    unsigned short lsb;
    unsigned char bits, up, es;
    signed char ret;
};
constexpr int kMaxSlots = 16;
template <int L>
struct PxLayout;
template <>
struct PxLayout<1> {  // 16-byte dual-return pixel: RNG19_RFL8_SIG16_NIR16_DUAL, ..._ZONE16_DUAL
    static constexpr int cds = 16, n = 10;
    static constexpr PxSlot s[n] = {{0, 19, 0, 4, 0},  {19, 5, 0, 1, -1},  {24, 8, 0, 1, -1}, {32, 19, 0, 4, 1},
                                    {51, 5, 0, 1, -1}, {56, 8, 0, 1, -1},  {64, 16, 0, 2, -1}, {80, 16, 0, 2, -1},
                                    {96, 16, 0, 2, -1}, {120, 8, 0, 1, -1}};
};
template <>
struct PxLayout<2> {  // 12-byte single-return pixel: RNG19_RFL8_SIG16_NIR16 (+ _ZONE16)
    static constexpr int cds = 12, n = 8;
    static constexpr PxSlot s[n] = {{0, 19, 0, 4, 0},   {19, 5, 0, 1, -1},  {32, 8, 0, 1, -1}, {40, 8, 0, 1, -1},
                                    {48, 16, 0, 2, -1}, {64, 16, 0, 2, -1}, {80, 16, 0, 2, -1}, {88, 8, 0, 1, -1}};
};
template <>
struct PxLayout<3> {  // 4-byte low-data-rate pixel: RNG15_RFL8_NIR8, RNG15_RFL8_WIN8
    static constexpr int cds = 4, n = 5;
    static constexpr PxSlot s[n] = {{0, 15, 3, 4, 0}, {15, 1, 0, 1, -1}, {16, 8, 0, 1, -1}, {24, 8, 4, 2, -1},
                                    {24, 8, 0, 1, -1}};
};
template <>
struct PxLayout<4> {  // 8-byte low-data-rate dual pixel: (FUSA_)RNG15_RFL8_NIR8_DUAL, RNG15_RFL8_NIR8_ZONE16
    static constexpr int cds = 8, n = 9;
    static constexpr PxSlot s[n] = {{0, 15, 3, 4, 0},  {15, 1, 0, 1, -1}, {16, 8, 0, 1, -1}, {24, 8, 4, 2, -1},
                                    {32, 15, 3, 4, 1}, {47, 1, 0, 1, -1}, {48, 8, 0, 1, -1}, {56, 8, 0, 1, -1},
                                    {32, 16, 0, 2, -1}};
};
template <>
struct PxLayout<5> {  // LEGACY 12-byte pixel
    static constexpr int cds = 12, n = 5;
    static constexpr PxSlot s[n] = {{0, 20, 0, 4, 0}, {28, 4, 0, 1, -1}, {32, 8, 0, 1, -1}, {48, 16, 0, 2, -1},
                                    {64, 16, 0, 2, -1}};
};

template <int L, int I>
__device__ __forceinline__ uint32_t slot_value(const uint32_t (&w)[PxLayout<L>::cds / 4]) {
    constexpr PxSlot sl = PxLayout<L>::s[I];
    constexpr int wi = sl.lsb / 32, bo = sl.lsb % 32;
    constexpr uint32_t mask = sl.bits >= 32 ? 0xffffffffu : ((1u << sl.bits) - 1u);
    uint32_t v;
    if constexpr (bo + sl.bits <= 32) {
        v = w[wi];
        if constexpr (bo != 0) v >>= bo;
        if constexpr (bo + sl.bits != 32) v &= mask;
    } else {
        v = __funnelshift_r(w[wi], w[wi + 1], bo) & mask;
    }
    if constexpr (sl.up != 0) v <<= sl.up;
    return v;
}

// ALL (output mode of a tile, uniform): 1 = every slot of the layout has an output image and every range slot a
// destaggered image (the default LidarFrame of the profile with a fused cloud), 2 = every slot has an output
// image and there is no destaggered range (the plain ScanBatcher result) -- no null tests in the row loop
// either way; 0 = anything else, tested pointer by pointer.
// (the default LidarFrame of the profile with a fused cloud) -> no null tests in the row loop.
template <int L, int I, bool FULL, int ALL>
__device__ __forceinline__ void slot_store(const uint32_t (&w)[PxLayout<L>::cds / 4], uint8_t* const (&outp)[kMaxSlots],
                                           uint32_t* const (&rdp)[2], unsigned pix, unsigned rdpix,
                                           bool col_valid, bool lane_on) {
    constexpr PxSlot sl = PxLayout<L>::s[I];
    uint8_t* o = outp[I];
    uint32_t* r = nullptr;
    if constexpr (sl.ret >= 0) r = rdp[sl.ret];
    if (ALL != 0 || o != nullptr || r != nullptr) {  // uniform per tile
        uint32_t v = slot_value<L, I>(w);
        if (!FULL) v = col_valid ? v : 0u;
        if (FULL || lane_on) {
            if (ALL != 0 || o != nullptr) {
                __builtin_assume(__isGlobal(o));
#ifdef OB_K2_STREAM_STORES  // experiment (measured slower, 0.130 vs 0.113 ms): evict-first stores for the write-once outputs
                if constexpr (sl.es == 4) __stcs(reinterpret_cast<uint32_t*>(o) + pix, v);
                else if constexpr (sl.es == 2) __stcs(reinterpret_cast<unsigned short*>(o) + pix, static_cast<unsigned short>(v));
                else __stcs(reinterpret_cast<unsigned char*>(o) + pix, static_cast<unsigned char>(v));
#else
                if constexpr (sl.es == 4) reinterpret_cast<uint32_t*>(o)[pix] = v;
                else if constexpr (sl.es == 2) reinterpret_cast<uint16_t*>(o)[pix] = static_cast<uint16_t>(v);
                else o[pix] = static_cast<uint8_t>(v);
#endif
            }
            if constexpr (sl.ret >= 0) {
                if (ALL == 1 || (ALL == 0 && r != nullptr)) {
                    __builtin_assume(__isGlobal(r));
#ifdef OB_K2_STREAM_STORES
                    __stcs(r + rdpix, v);
#else
                    r[rdpix] = v;
#endif
                }
            }
        }
    }
}

template <int L, bool FULL, int ALL, int... I>
__device__ __forceinline__ void store_all(const uint32_t (&w)[PxLayout<L>::cds / 4], uint8_t* const (&outp)[kMaxSlots],
                                          uint32_t* const (&rdp)[2], unsigned pix, unsigned rdpix, bool col_valid,
                                          bool lane_on, std::integer_sequence<int, I...>) {
    (slot_store<L, I, FULL, ALL>(w, outp, rdp, pix, rdpix, col_valid, lane_on), ...);
}

// Phase A with a compile-time layout: lane = frame column, warps stride the rows, all fields of a
// pixel from registers.
template <int L, bool FULL, int ALL>
__device__ __forceinline__ void decode_static(const uint8_t* px0, bool col_valid, bool lane_on,
                                              uint8_t* const (&outp)[kMaxSlots], uint32_t* const (&rdp)[2],
                                              unsigned col, unsigned W, unsigned H, unsigned row0, unsigned rstep,
                                              const DecodeParams& p) {
    constexpr int NW = PxLayout<L>::cds / 4;
    const bool has_rd = ALL == 1 || (ALL == 0 && (rdp[0] != nullptr || rdp[1] != nullptr));
    const bool has_shift = p.has_shift != 0;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(px0) + row0 * NW;
    const unsigned wstep = rstep * NW;
    unsigned pix = row0 * W + col;
    const unsigned pstep = rstep * W;
#pragma unroll 2
    for (unsigned row = row0; row < H; row += rstep) {
        uint32_t w[NW];
#pragma unroll
        for (int i = 0; i < NW; ++i) w[i] = wp[i];
        unsigned rdpix = pix;
        if (has_rd) {
            unsigned dcol = col + (has_shift ? p.shift[row] : 0u);
            dcol = dcol >= W ? dcol - W : dcol;
            rdpix = pix - col + dcol;
        }
        store_all<L, FULL, ALL>(w, outp, rdp, pix, rdpix, col_valid, lane_on,
                                std::make_integer_sequence<int, PxLayout<L>::n>{});
        wp += wstep;
        pix += pstep;
    }
}

// The same row body with the LAST rows handed out dynamically: every warp first decodes `n_static` rows of its
// own residue class (row0 + i * rstep, no hand-out cost), then the warps share the remaining rows of the tile
// through a shared-memory counter, so that they finish a tile together whatever H modulo the warp count is
// (128 rows over 24 warps is 5.33 rows each: with a fixed stride the 6-row warps set the pace and the 5-row
// warps wait for the next tile's packets).  Handing out ALL rows that way costs one same-address atomic per
// row and warp -- 152 serialised shared-memory atomics per tile, a third of a tile's time when nothing else is
// going on (tools/k2_parts.py).  The ticket of the next row is drawn while the current one is decoded.
template <int L, bool FULL, int ALL>
__device__ __forceinline__ void decode_static_dyn(const uint8_t* px0, bool col_valid, bool lane_on,
                                                  uint8_t* const (&outp)[kMaxSlots], uint32_t* const (&rdp)[2],
                                                  unsigned col, unsigned W, unsigned H, unsigned* row_ctr,
                                                  unsigned row0, unsigned rstep, unsigned n_static,
                                                  const DecodeParams& p) {
    constexpr int NW = PxLayout<L>::cds / 4;
    const bool has_rd = ALL == 1 || (ALL == 0 && (rdp[0] != nullptr || rdp[1] != nullptr));
    const bool has_shift = p.has_shift != 0;
    const unsigned lane = threadIdx.x & 31u;
    auto one_row = [&](unsigned row) {
        const uint32_t* wp = reinterpret_cast<const uint32_t*>(px0) + row * NW;
        uint32_t w[NW];
#pragma unroll
        for (int i = 0; i < NW; ++i) w[i] = wp[i];
        const unsigned pix = row * W + col;
        unsigned rdpix = pix;
        if (has_rd) {
            unsigned dcol = col + (has_shift ? p.shift[row] : 0u);
            dcol = dcol >= W ? dcol - W : dcol;
            rdpix = pix - col + dcol;
        }
        store_all<L, FULL, ALL>(w, outp, rdp, pix, rdpix, col_valid, lane_on,
                                std::make_integer_sequence<int, PxLayout<L>::n>{});
    };
    for (unsigned i = 0; i < n_static; ++i) one_row(row0 + i * rstep);
    const unsigned base = n_static * rstep;  // first dynamically assigned row
    if (base >= H) return;
    unsigned nxt = 0;
    if (lane == 0) nxt = atomicAdd(row_ctr, 1u);
    for (;;) {
        const unsigned row = base + __shfl_sync(0xffffffffu, nxt, 0);
        if (row >= H) break;
        if (lane == 0) nxt = atomicAdd(row_ctr, 1u);
        one_row(row);
    }
}

// output mode of a tile for the compile-time layouts (see slot_store)
__device__ __forceinline__ int static_output_mode(const DecodeParams& p, const DecodeFrame& fr) {
    if (p.layout_all == 0 || (fr.flags & kFrameAllFields) == 0 || p.n_returns == 0) return 0;
    const bool rd0 = fr.rd[0] != nullptr, rd1 = p.n_returns > 1 ? fr.rd[1] != nullptr : rd0;
    if (rd0 && rd1) return 1;
    if (!rd0 && !(p.n_returns > 1 && fr.rd[1] != nullptr)) return 2;
    return 0;
}

template <int L>
__device__ __forceinline__ void decode_static_tile_dyn(bool full, int all, const uint8_t* px0, bool col_valid,
                                                       bool lane_on, uint8_t* const (&outp)[kMaxSlots],
                                                       uint32_t* const (&rdp)[2], unsigned col, unsigned W,
                                                       unsigned H, unsigned* row_ctr, unsigned row0, unsigned rstep,
                                                       unsigned n_static, const DecodeParams& p) {
    if (full && all == 1) decode_static_dyn<L, true, 1>(px0, true, true, outp, rdp, col, W, H, row_ctr, row0, rstep, n_static, p);
    else if (full && all == 2) decode_static_dyn<L, true, 2>(px0, true, true, outp, rdp, col, W, H, row_ctr, row0, rstep, n_static, p);
    else if (full) decode_static_dyn<L, true, 0>(px0, true, true, outp, rdp, col, W, H, row_ctr, row0, rstep, n_static, p);
    else decode_static_dyn<L, false, 0>(px0, col_valid, lane_on, outp, rdp, col, W, H, row_ctr, row0, rstep, n_static, p);
}

template <int L>
__device__ __forceinline__ void decode_static_tile(bool full, int all, const uint8_t* px0, bool col_valid,
                                                   bool lane_on, uint8_t* const (&outp)[kMaxSlots],
                                                   uint32_t* const (&rdp)[2], unsigned col, unsigned W, unsigned H,
                                                   unsigned row0, unsigned rstep, const DecodeParams& p) {
    if (full && all == 1) decode_static<L, true, 1>(px0, true, true, outp, rdp, col, W, H, row0, rstep, p);
    else if (full && all == 2) decode_static<L, true, 2>(px0, true, true, outp, rdp, col, W, H, row0, rstep, p);
    else if (full) decode_static<L, true, 0>(px0, true, true, outp, rdp, col, W, H, row0, rstep, p);
    else decode_static<L, false, 0>(px0, col_valid, lane_on, outp, rdp, col, W, H, row0, rstep, p);
}

}  // namespace ob
