// ob_encode.cu -- K4: LidarFrame fields -> lidar UDP packets on the device (the inverse of K2), with the
// CRC64 of the standard packet footer.  SURVEY 8f-3 (GPU-side frame_to_packets / set_block + CRC64).
//
// What it replaces (reference paths relative to /root/reference):
//   impl::frame_to_packets (lidar part)   ouster_core/include/ouster/core/impl/lidar_frame_impl.h:435-531
//   PacketFormat::set_block<T>            ouster_core/src/parsing.cpp:1056-1090
//   FieldDecodeInfo::set<T>               ouster_core/include/ouster/core/field_decode_info.h:64-78
//   crc64_compute / calculate_crc         ouster_core/src/parsing.cpp:1183-1234
//
// One CTA builds one packet in shared memory: the packet header bytes come from the host (frame id,
// init id, serial number, alert flags ... -- 32 bytes per packet, written with the reference's own
// setters), the column headers from the frame's per-column arrays, and every thread packs the channel
// data block of one pixel at a time, for the columns whose status has bit 0 set (set_block skips the
// others).  Every field is written as FieldDecodeInfo::set writes it: value << shift (or >> -shift),
// & mask, then the mask's bits of the 8-byte window at the field's byte offset are cleared and the value
// OR-ed in -- zero values included.  The pixel's thread takes the fields in decoder (PacketFormat) order,
// so where masks overlap (FIVE_WORD_PIXEL's RAW32 words and the named fields they cover) the last field
// decides the bits, as in the reference.  That needs every mask inside its own pixel's bytes, which
// ob_encode_frames checks: threads of neighbouring pixels then touch disjoint bits of a shared word, and
// the shared-memory atomics make the order between them irrelevant.
// The CRC is ECMA-182 reflected (poly 0xC96C5795D7870F42, init ~0, final ~): the packet is cut into 256
// equal chunks whose init-0 CRCs are computed by 256 threads with the Sarwate byte table, merged pairwise
// with precomputed GF(2) "advance by N bytes" matrices (CRC is linear over GF(2)), and corrected for the
// non-zero initial register by one constant.
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "ob_api_common.h"
#include "ob_encode.h"

namespace ob {

namespace {

constexpr int kEncThreads = 256;
constexpr uint64_t kCrcPoly = 0xC96C5795D7870F42ull;

struct CrcTables {  // device memory, shared by every encoder with the same chunk length
    uint64_t byte_table[256];
    uint64_t advance[8][64];  // advance[k]: matrix (64 columns) of "append chunk_bytes * 2^k zero bytes"
    uint64_t init_term;       // contribution of the initial register ~0 after `crc_len` bytes
    uint32_t chunk_bytes;     // multiple of 4 with an odd word count (conflict-free strided reads)
    uint32_t crc_len;         // bytes covered by the CRC (packet_size - 8)
};

struct EncodeParams {
    DecodeLayout L;
    const EncodeFrame* frames;
    const CrcTables* crc;
    uint32_t n_packets_per_frame;
    uint32_t with_crc;
};

__device__ __forceinline__ uint64_t load_elem(const void* base, size_t idx, uint32_t es) {
    switch (es) {
        case 1: return static_cast<const uint8_t*>(base)[idx];
        case 2: return static_cast<const uint16_t*>(base)[idx];
        case 4: return static_cast<const uint32_t*>(base)[idx];
        case 8: return static_cast<const uint64_t*>(base)[idx];
        default: {  // 6 bytes: 3 x 16 bit
            const uint16_t* q = static_cast<const uint16_t*>(base) + idx * 3;
            return static_cast<uint64_t>(q[0]) | (static_cast<uint64_t>(q[1]) << 16) | (static_cast<uint64_t>(q[2]) << 32);
        }
    }
}

// the 64-bit value `v` placed at byte `sh / 8` of three consecutive 32-bit words
__device__ __forceinline__ void split_window(uint64_t v, uint32_t sh, uint32_t out[3]) {
    const uint32_t lo = static_cast<uint32_t>(v), hi = static_cast<uint32_t>(v >> 32);
    out[0] = lo << sh;
    out[1] = sh ? ((lo >> (32u - sh)) | (hi << sh)) : hi;
    out[2] = sh ? (hi >> (32u - sh)) : 0u;
}

// FieldDecodeInfo::set (field_decode_info.h:64-78) on the 8-byte window at `byte_off`: clear the bits of
// f.mask, then OR in value << shift (>> -shift) & mask.  Bits outside the mask are left alone.
__device__ __forceinline__ void set_field(uint32_t* words, uint32_t n_words, uint32_t byte_off, const DecodeField& f,
                                          uint64_t v) {
    if (f.shift > 0) v <<= f.shift;
    else if (f.shift < 0) v >>= -f.shift;
    const uint32_t wi = byte_off >> 2, sh = (byte_off & 3u) * 8u;
    uint32_t m[3], w[3];
    split_window(f.mask, sh, m);
    split_window(v & f.mask, sh, w);
#pragma unroll
    for (uint32_t j = 0; j < 3; ++j) {
        if (m[j] == 0u || wi + j >= n_words) continue;
        atomicAnd(&words[wi + j], ~m[j]);
        if (w[j]) atomicOr(&words[wi + j], w[j]);
    }
}

__device__ __forceinline__ uint64_t gf2_apply(const uint64_t* cols, uint64_t v) {
    uint64_t r = 0;
#pragma unroll 8
    for (int j = 0; j < 64; ++j) r ^= ((v >> j) & 1ull) ? cols[j] : 0ull;
    return r;
}

__global__ void __launch_bounds__(kEncThreads) encode_kernel(const __grid_constant__ EncodeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const DecodeLayout& L = p.L;
    uint32_t* words = reinterpret_cast<uint32_t*>(smem);
    const uint32_t n_words = (L.packet_size + 3u) / 4u + 2u;  // + slack for trailing 8-byte windows
    uint64_t* partial = reinterpret_cast<uint64_t*>(smem + ((static_cast<size_t>(n_words) * 4u + 7u) & ~static_cast<size_t>(7)));
    uint64_t* table = partial + kEncThreads;
    const int tid = threadIdx.x;
    const uint32_t f = blockIdx.x / p.n_packets_per_frame, pk = blockIdx.x - f * p.n_packets_per_frame;
    const EncodeFrame& fr = p.frames[f];

    for (uint32_t i = tid; i < n_words; i += kEncThreads) words[i] = 0u;
    if (p.with_crc)
        for (int i = tid; i < 256; i += kEncThreads) table[i] = p.crc->byte_table[i];
    __syncthreads();

    // ---- packet header (host-built bytes) and column headers ----
    if (fr.packet_headers != nullptr) {
        const uint32_t hb = min(fr.header_bytes, L.packet_size);
        for (uint32_t i = tid; i < hb; i += kEncThreads) smem[i] = fr.packet_headers[static_cast<size_t>(pk) * fr.header_bytes + i];
    }
    __syncthreads();
    for (uint32_t c = tid; c < L.cpp; c += kEncThreads) {
        const uint32_t id = pk * L.cpp + c;
        const uint32_t col0 = L.packet_header_size + c * L.col_size;
        const uint64_t st = fr.status ? fr.status[id] : 0u;
        const uint64_t ts = fr.timestamp ? fr.timestamp[id] : 0u;
        set_field(words, n_words, col0 + L.status.offset, L.status, st);
        set_field(words, n_words, col0 + L.mid.offset, L.mid, id & 0xffffu);
        set_field(words, n_words, col0 + L.ts.offset, L.ts, ts);
    }

    // ---- channel data: one pixel per thread and trip; set_block skips columns without status bit 0 ----
    const uint32_t n_px = L.cpp * L.H;
    for (uint32_t i = tid; i < n_px; i += kEncThreads) {
        const uint32_t c = i % L.cpp, row = i / L.cpp;  // lanes walk the columns: coalesced image reads
        const uint32_t id = pk * L.cpp + c;
        if (!(fr.status && (fr.status[id] & 1u))) continue;
        const uint32_t px0 = L.packet_header_size + c * L.col_size + L.col_header_size + row * L.channel_data_size;
        const size_t src = static_cast<size_t>(row) * L.W + id;
        for (uint32_t k = 0; k < L.n_fields; ++k) {
            if (fr.fields[k] == nullptr) continue;
            const DecodeField& fd = L.fields[k];
            set_field(words, n_words, px0 + fd.offset, fd, load_elem(fr.fields[k], src, fd.elem_size));
        }
    }
    __syncthreads();

    // ---- CRC64 over packet_size - 8 bytes, written little-endian into the last 8 bytes ----
    if (p.with_crc) {
        const CrcTables& ct = *p.crc;
        const uint32_t cb = ct.chunk_bytes, n = ct.crc_len;
        const uint32_t pad = cb * kEncThreads - n;  // virtual leading zero bytes (neutral with init 0)
        // chunk `tid` covers padded bytes [tid*cb, (tid+1)*cb) = real bytes [tid*cb - pad, ...)
        uint64_t crc = 0;
        const long long start = static_cast<long long>(tid) * cb - pad;
        for (uint32_t b = 0; b < cb; ++b) {
            const long long a = start + b;
            if (a < 0) continue;
            crc = table[(smem[a] ^ crc) & 0xffu] ^ (crc >> 8);
        }
        partial[tid] = crc;
        __syncthreads();
        // pairwise merge: crc(A || B) = advance(crc(A), |B|) ^ crc(B), |B| = cb << k at level k
        for (int k = 0, step = 1; step < kEncThreads; ++k, step <<= 1) {
            if ((tid & (2 * step - 1)) == 0) partial[tid] = gf2_apply(ct.advance[k], partial[tid]) ^ partial[tid + step];
            __syncthreads();
        }
        if (tid == 0) {
            const uint64_t v = ~(partial[0] ^ ct.init_term);
            words[(L.packet_size - 8u) / 4u] = static_cast<uint32_t>(v);       // packet_size % 4 == 0 (checked on the host)
            words[(L.packet_size - 8u) / 4u + 1u] = static_cast<uint32_t>(v >> 32);
        }
        __syncthreads();
    }

    // ---- out ----
    uint8_t* dst = fr.packets + static_cast<size_t>(pk) * fr.packet_stride;
    if ((reinterpret_cast<uintptr_t>(dst) & 3u) == 0 && (L.packet_size & 3u) == 0) {
        uint32_t* d4 = reinterpret_cast<uint32_t*>(dst);
        for (uint32_t i = tid; i < L.packet_size / 4u; i += kEncThreads) d4[i] = words[i];
    } else {
        for (uint32_t i = tid; i < L.packet_size; i += kEncThreads) dst[i] = smem[i];
    }
}

// ---- host: CRC tables (Sarwate byte table, advance matrices, init term) ----
uint64_t crc_byte(uint64_t crc, const uint64_t* table, uint8_t b) { return table[(b ^ crc) & 0xff] ^ (crc >> 8); }

void build_byte_table(uint64_t* t) {  // parsing.cpp:1187-1203
    for (uint32_t i = 0; i < 256; ++i) {
        uint64_t r = i;
        for (int j = 0; j < 8; ++j) r = (r >> 1) ^ (kCrcPoly & ~((r & 1) - 1));
        t[i] = r;
    }
}

// columns of the linear map "register after appending one zero byte"
void zero_byte_matrix(const uint64_t* table, uint64_t* cols) {
    for (int j = 0; j < 64; ++j) cols[j] = crc_byte(1ull << j, table, 0);
}
uint64_t apply(const uint64_t* cols, uint64_t v) {
    uint64_t r = 0;
    for (int j = 0; j < 64; ++j)
        if ((v >> j) & 1ull) r ^= cols[j];
    return r;
}
void mat_mul(const uint64_t* a, const uint64_t* b, uint64_t* out) {  // out = a o b (apply b first)
    for (int j = 0; j < 64; ++j) out[j] = apply(a, b[j]);
}
void mat_pow(const uint64_t* base, uint64_t n, uint64_t* out) {
    uint64_t sq[64], acc[64], tmp[64];
    for (int j = 0; j < 64; ++j) {
        acc[j] = 1ull << j;
        sq[j] = base[j];
    }
    while (n) {
        if (n & 1) {
            mat_mul(sq, acc, tmp);
            std::memcpy(acc, tmp, sizeof(acc));
        }
        mat_mul(sq, sq, tmp);
        std::memcpy(sq, tmp, sizeof(sq));
        n >>= 1;
    }
    std::memcpy(out, acc, sizeof(acc));
}

std::mutex g_crc_mx;
std::vector<std::pair<std::pair<int, uint32_t>, CrcTables*>> g_crc_tables;  // (device, crc_len) -> device tables

const CrcTables* crc_tables_for(int device, uint32_t crc_len) {
    std::lock_guard<std::mutex> lk(g_crc_mx);
    for (auto& e : g_crc_tables)
        if (e.first.first == device && e.first.second == crc_len) return e.second;
    auto h = std::make_unique<CrcTables>();
    build_byte_table(h->byte_table);
    uint32_t cb = (crc_len + kEncThreads - 1) / kEncThreads;
    cb = (cb + 3u) & ~3u;
    if (((cb / 4u) & 1u) == 0) cb += 4u;  // odd word count: threads hit distinct banks
    h->chunk_bytes = cb;
    h->crc_len = crc_len;
    uint64_t z[64], m[64];
    zero_byte_matrix(h->byte_table, z);
    for (int k = 0; k < 8; ++k) {
        mat_pow(z, static_cast<uint64_t>(cb) << k, m);
        std::memcpy(h->advance[k], m, sizeof(m));
    }
    mat_pow(z, crc_len, m);
    h->init_term = apply(m, ~0ull);
    CrcTables* d = nullptr;
    if (cudaMalloc(&d, sizeof(CrcTables)) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    if (cudaMemcpy(d, h.get(), sizeof(CrcTables), cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaGetLastError();
        cudaFree(d);
        return nullptr;
    }
    g_crc_tables.push_back({{device, crc_len}, d});
    return d;
}

}  // namespace

cudaError_t launch_encode(const DecodeLayout& L, const EncodeFrame* frames_dev, uint32_t n_frames, bool with_crc,
                          int device, cudaStream_t st) {
    if (n_frames == 0) return cudaSuccess;
    if (L.cpp == 0 || L.W % L.cpp != 0 || L.packet_size < 8) return cudaErrorInvalidValue;
    EncodeParams p;
    p.L = L;
    p.frames = frames_dev;
    p.n_packets_per_frame = L.W / L.cpp;
    p.with_crc = with_crc ? 1u : 0u;
    p.crc = nullptr;
    if (with_crc) {
        if (L.packet_size % 4 != 0) return cudaErrorInvalidValue;
        p.crc = crc_tables_for(device, L.packet_size - 8);
        if (!p.crc) return cudaErrorMemoryAllocation;
    }
    const size_t n_words = (L.packet_size + 3u) / 4u + 2u;
    const size_t smem = ((n_words * 4 + 7) & ~static_cast<size_t>(7)) + (kEncThreads + 256) * sizeof(uint64_t);
    if (smem > 227 * 1024) return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    launch(OB_FAM_ENCODE, encode_kernel, n_frames * p.n_packets_per_frame, kEncThreads, smem, st, p);
    return cudaGetLastError();
}

}  // namespace ob
