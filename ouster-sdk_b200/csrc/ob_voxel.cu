// ob_voxel.cu -- voxel-grid downsampling (SURVEY 8f-2): the reference's sequential hash-map insertion
// restated as a sort-based data-parallel pipeline.
//
// What it replaces (reference paths relative to the reference tree, ouster-sdk 1.0.1):
//   core::voxel_downsample                   ouster_core/src/voxel_hash_map.cpp:262-310
//   core::voxel_downsample_3d / _xd          ouster_core/src/voxel_hash_map.cpp:312-393
//   insertion strategies, PointNormalBucket  ouster_core/include/ouster/core/voxel_hash_map.h:142-185, 287-334, 587-635
//   algorithm::voxel_downsample_with_normals ouster_algorithm/src/voxel_downsample.cpp:21-57
//
// The reference inserts the points one at a time into a tsl::robin_map.  Every result only depends on
// which points share a voxel and on their order inside the voxel, so here:
//   1. key      one thread per point: the three int32 voxel coordinates (padding rows sort last);
//   2. sort     stable radix sort of (key, sequence position) -- CUB, header-only in the CUDA toolkit;
//   3. segments a head flag per voxel, written at the head's sequence position; an inclusive scan of it
//               in sequence order numbers the voxels by first appearance without another sort;
//   4. reduce   one thread per voxel walks its points in sequence order (sequential sums: bit-exact
//               AVERAGE; greedy FIRST_N; RANDOM with its global RNG stream, see below);
//   5. emit     a scan of the per-voxel output counts places every voxel's rows.
// RANDOM: the reference draws one xorshift32 number (seed 42) per insertion into a full bucket, in input
// order.  The k-th such insertion gets state M^(k+1)*42, M the 32x32 GF(2) matrix of one xorshift step;
// k comes from an exclusive scan of the "bucket full" flags, M^(2^b) are compile-time jump matrices.
// SHUFFLE_FIRST (core::voxel_downsample): the Fisher-Yates shuffle depends only on n; its permutation is
// resolved without a serial loop (DESIGN 4, f-5), then the shuffled sequence goes through FIRST_N with
// one slot per voxel.
#include <algorithm>

#include "ob_api_common.h"
#include "ob_cub.cuh"
#include "ob_rows.cuh"
#include "ob_voxel_common.cuh"

namespace ob {

namespace {

// ---- xorshift32 jump matrices ----
struct JumpTable {
    uint32_t m[32][32];  // m[b][j]: column j of M^(2^b), i.e. the image of the basis vector 1 << j
};

constexpr uint32_t xs_step(uint32_t s) {
    s ^= s << 13;
    s ^= s >> 17;
    s ^= s << 5;
    return s;
}

constexpr uint32_t gf2_apply(const uint32_t (&cols)[32], uint32_t v) {
    uint32_t r = 0;
    for (int j = 0; j < 32; ++j)
        if ((v >> j) & 1u) r ^= cols[j];
    return r;
}

constexpr JumpTable make_jump_table() {
    JumpTable t{};
    for (int j = 0; j < 32; ++j) t.m[0][j] = xs_step(1u << j);
    for (int b = 1; b < 32; ++b)
        for (int j = 0; j < 32; ++j) t.m[b][j] = gf2_apply(t.m[b - 1], t.m[b - 1][j]);
    return t;
}

__constant__ JumpTable kJump = make_jump_table();

// state of the reference's xorshift32 after `steps` steps from seed 42
__device__ uint32_t xs_state_after(unsigned long long steps) {
    uint32_t v = 42u;
    for (int b = 0; steps != 0; ++b, steps >>= 1) {
        if (steps & 1ull) {
            uint32_t r = 0;
#pragma unroll 8
            for (int j = 0; j < 32; ++j)
                if ((v >> j) & 1u) r ^= kJump.m[b][j];
            v = r;
        }
    }
    return v;
}

struct VoxelParams {
    const void* points;   // capacity x cols of T
    const void* normals;  // POINT_NORMAL: capacity x 3 of T
    const unsigned long long* n_dev;  // device count, or null: n_host
    unsigned long long n_host;
    unsigned cap, cols;
    int mode;
    double inv;           // 1.0 / voxel_size
    double res_sq;        // voxel_size^2 / max_points_per_voxel (first_n_point)
    unsigned long long max_pts;
    unsigned long long min_pts;
    const uint32_t* order;  // sequence position -> input row (SHUFFLE_FIRST), null = identity
};

__device__ __forceinline__ unsigned n_of(const VoxelParams& p) {
    if (p.n_dev == nullptr) return static_cast<unsigned>(p.n_host);
    const unsigned long long n = *p.n_dev;
    return n < p.cap ? static_cast<unsigned>(n) : p.cap;
}

template <typename T>
__device__ __forceinline__ double ld(const void* base, size_t i) {
    return static_cast<double>(static_cast<const T*>(base)[i]);
}

// ---- Fisher-Yates without the serial loop (SHUFFLE_FIRST) ----
// step s < n-1 swaps positions s and j_s = s + ((u64)rand_s * (n - s)) >> 32, rand_s the (s+1)-th draw;
// step n-1 is treated as j = n-1.  Padding steps get the key `cap` (sorts last).
__global__ void vx_shuffle_draw_kernel(VoxelParams p, uint32_t* jkey, uint32_t* step) {
    const unsigned s = tid_global();
    if (s >= p.cap) return;
    const unsigned n = n_of(p);
    uint32_t j = p.cap;
    if (s + 1 < n) {
        const unsigned long long r = xs_state_after(static_cast<unsigned long long>(s) + 1ull);
        j = s + static_cast<uint32_t>((r * static_cast<unsigned long long>(n - s)) >> 32);
    } else if (s + 1 == n) {
        j = s;
    }
    jkey[s] = j;
    step[s] = s;
}

// over the steps sorted by (j, s): where each step landed, and the last sorted slot of every j
__global__ void vx_shuffle_index_kernel(unsigned cap, const uint32_t* sj, const uint32_t* ss, uint32_t* where,
                                        int32_t* last_of) {
    const unsigned q = tid_global();
    if (q >= cap) return;
    const uint32_t j = sj[q];
    if (j >= cap) return;
    where[ss[q]] = q;
    if (q + 1 == cap || sj[q + 1] != j) last_of[j] = static_cast<int32_t>(q);
}

// the element that ends at position i: f(pred(i)) when an earlier step chose the same j, else j_i, with
// f(p) = p unless an earlier step s < p chose j_s = p, then f(L(p)), L(p) the last such step
__global__ void vx_shuffle_perm_kernel(VoxelParams p, const uint32_t* sj, const uint32_t* ss, const uint32_t* where,
                                       const int32_t* last_of, uint32_t* order) {
    const unsigned i = tid_global();
    if (i >= p.cap) return;
    const unsigned n = n_of(p);
    if (i >= n) {
        order[i] = i;
        return;
    }
    const unsigned q = where[i];
    if (q == 0 || sj[q - 1] != sj[q]) {
        order[i] = sj[q];
        return;
    }
    uint32_t e = ss[q - 1];
    for (;;) {
        int32_t ql = last_of[e];
        if (ql < 0) break;
        uint32_t s = ss[ql];
        if (s == e) {  // step e itself chose j = e; the one before it in the group is L(e)
            if (ql == 0 || sj[ql - 1] != e) break;
            s = ss[ql - 1];
        }
        e = s;
    }
    order[i] = e;
}

// ---- 1. keys ----
template <typename T>
__global__ void vx_key_kernel(VoxelParams p, VKey* keys, uint32_t* seq) {
    const unsigned t = tid_global();
    if (t >= p.cap) return;
    VKey k{1u, 0, 0, 0};
    if (t < n_of(p)) {
        const size_t row = p.order ? p.order[t] : t;
        const double x = ld<T>(p.points, row * p.cols), y = ld<T>(p.points, row * p.cols + 1),
                     z = ld<T>(p.points, row * p.cols + 2);
        bool ok = true;
        if (p.mode == OB_VOXEL_POINT_NORMAL) {  // voxel_downsample.cpp:40-42
            const double a = ld<T>(p.normals, row * 3), b = ld<T>(p.normals, row * 3 + 1), c = ld<T>(p.normals, row * 3 + 2);
            ok = finite3(x, y, z) && finite3(a, b, c) && sqrt(sqn3(a, b, c)) > 1e-12;
        }
        if (ok)
            k = VKey{0u, floor_cast<int32_t>(mul(x, p.inv)), floor_cast<int32_t>(mul(y, p.inv)),
                     floor_cast<int32_t>(mul(z, p.inv))};
    }
    keys[t] = k;
    seq[t] = t;
}

// ---- 3. segments (vx_head_kernel, vx_seg_kernel, segment_end: ob_voxel_common.cuh) ----
struct Seg {
    unsigned start, len;
};
// the same search as segment_end, backwards: the first sorted position of the voxel that holds position q
__device__ __forceinline__ unsigned segment_begin(unsigned q, const VKey* sk) {
    const VKey k = sk[q];
    unsigned first = q, step = 1;
    int lo = -1;
    for (;;) {
        if (step > first || !same_key(sk[first - step], k)) {
            lo = step > first ? -1 : static_cast<int>(first - step);
            break;
        }
        first -= step;
        step <<= 1;
    }
    while (static_cast<int>(first) - lo > 1) {
        const unsigned mid = static_cast<unsigned>(lo + (static_cast<int>(first) - lo) / 2);
        if (same_key(sk[mid], k)) first = mid;
        else lo = static_cast<int>(mid);
    }
    return first;
}
__device__ __forceinline__ Seg segment_of(unsigned r, unsigned cap, const VKey* sk, const uint32_t* seg_start) {
    Seg s;
    s.start = seg_start[r];
    s.len = segment_end(s.start, cap, sk) - s.start;
    return s;
}

__device__ __forceinline__ uint32_t row_of(const VoxelParams& p, const uint32_t* sseq, unsigned q) {
    const uint32_t t = sseq[q];
    return p.order ? p.order[t] : t;
}

struct Work {
    const VKey* sk;
    const uint32_t* sseq;
    const uint32_t* vrank;     // inclusive scan of the head flags; vrank[cap-1] = number of voxels
    const uint32_t* seg_start; // per voxel (first-appearance rank): sorted position of its first point
    uint32_t* cnt;             // per voxel: rows it emits
    uint32_t* slot;            // sorted-position space: slot k of voxel r at slot[start + k] (input rows)
    double* vres;              // AVERAGE: cap x cols, POINT_NORMAL: cap x 6 (per voxel rank)
    uint32_t* vfirst;          // per voxel: input row of its first point
    uint32_t* full;            // RANDOM: 1 where the point's voxel already holds max points (sequence order)
    const uint32_t* draw;      // RANDOM: exclusive scan of `full` = the point's draw index
};

// A voxel's points are read kBatch at a time (all loads issued before the first use) and then consumed in
// input order: the sums stay sequential, the memory latency is paid once per batch.
constexpr unsigned kBatch = 8;

// ---- 4. per-voxel reductions ----
// AVERAGE_POINT (accumulate_strategy + AveragePointBucket) and POINT_NORMAL (PointNormalBucket): sums in
// input order starting from +0.0, then one division -- the reference's arithmetic, hence bit-exact.
template <typename T>
__global__ void vx_reduce_sum_kernel(VoxelParams p, Work w) {
    const unsigned r = tid_global();
    if (r >= p.cap) return;
    const unsigned nv = w.vrank[p.cap - 1];
    if (r >= nv) {
        w.cnt[r] = 0;
        return;
    }
    const Seg sg = segment_of(r, p.cap, w.sk, w.seg_start);
    const unsigned end = sg.start + sg.len;
    w.vfirst[r] = row_of(p, w.sseq, sg.start);
    const double cnt_d = static_cast<double>(sg.len);
    if (p.mode == OB_VOXEL_AVERAGE_POINT) {
        double* out = w.vres + static_cast<size_t>(r) * p.cols;
        for (unsigned c0 = 0; c0 < p.cols; c0 += 4) {
            double acc[4] = {0.0, 0.0, 0.0, 0.0};
            const unsigned nc = min(4u, p.cols - c0);
            for (unsigned q = sg.start; q < end; q += kBatch) {
                double v[kBatch][4];
#pragma unroll
                for (unsigned i = 0; i < kBatch; ++i) {
                    const size_t base = q + i < end ? static_cast<size_t>(row_of(p, w.sseq, q + i)) * p.cols + c0 : 0;
#pragma unroll
                    for (unsigned c = 0; c < 4; ++c) v[i][c] = (q + i < end && c < nc) ? ld<T>(p.points, base + c) : 0.0;
                }
#pragma unroll
                for (unsigned i = 0; i < kBatch; ++i)
                    if (q + i < end)
#pragma unroll
                        for (unsigned c = 0; c < 4; ++c) acc[c] = add(acc[c], v[i][c]);
            }
            for (unsigned c = 0; c < nc; ++c) out[c0 + c] = acc[c] / cnt_d;
        }
        w.cnt[r] = sg.len >= p.min_pts ? 1u : 0u;
        return;
    }
    // POINT_NORMAL: voxel_downsample.cpp:38-47, voxel_hash_map.h:164-175
    double ps[3] = {0.0, 0.0, 0.0}, ns[3] = {0.0, 0.0, 0.0};
    for (unsigned q = sg.start; q < end; q += kBatch) {
        double v[kBatch][6];
#pragma unroll
        for (unsigned i = 0; i < kBatch; ++i) {
            const size_t row = q + i < end ? row_of(p, w.sseq, q + i) : 0;
#pragma unroll
            for (unsigned c = 0; c < 3; ++c) {
                v[i][c] = q + i < end ? ld<T>(p.points, row * 3 + c) : 0.0;
                v[i][3 + c] = q + i < end ? ld<T>(p.normals, row * 3 + c) : 0.0;
            }
        }
#pragma unroll
        for (unsigned i = 0; i < kBatch; ++i) {
            if (q + i >= end) break;
            const double len = sqrt(sqn3(v[i][3], v[i][4], v[i][5]));
#pragma unroll
            for (unsigned c = 0; c < 3; ++c) {
                ps[c] = add(ps[c], v[i][c]);
                ns[c] = add(ns[c], v[i][3 + c] / len);
            }
        }
    }
    const double nl = sqrt(sqn3(ns[0], ns[1], ns[2]));
    double* out = w.vres + static_cast<size_t>(r) * 6;
    for (int c = 0; c < 3; ++c) {
        out[c] = ps[c] / cnt_d;
        out[3 + c] = ns[c] / nl;
    }
    w.cnt[r] = nl > 1e-12 ? 1u : 0u;
}

// FIRST_N_POINT (first_n_point, voxel_hash_map.h:287-301) and SHUFFLE_FIRST (max 1): greedy in input order,
// done once the voxel holds max points
template <typename T>
__global__ void vx_reduce_first_kernel(VoxelParams p, Work w) {
    const unsigned r = tid_global();
    if (r >= p.cap) return;
    const unsigned nv = w.vrank[p.cap - 1];
    if (r >= nv) {
        w.cnt[r] = 0;
        return;
    }
    const Seg sg = segment_of(r, p.cap, w.sk, w.seg_start);
    const unsigned end = sg.start + sg.len;
    uint32_t* b = w.slot + sg.start;
    unsigned fill = 0;
    for (unsigned q = sg.start; q < end && fill < p.max_pts; q += kBatch) {
        uint32_t rows[kBatch];
        double v[kBatch][3];
#pragma unroll
        for (unsigned i = 0; i < kBatch; ++i) {
            rows[i] = q + i < end ? row_of(p, w.sseq, q + i) : 0u;
#pragma unroll
            for (unsigned c = 0; c < 3; ++c) v[i][c] = q + i < end ? ld<T>(p.points, static_cast<size_t>(rows[i]) * p.cols + c) : 0.0;
        }
        for (unsigned i = 0; i < kBatch && q + i < end && fill < p.max_pts; ++i) {
            bool near = false;
            for (unsigned k = 0; k < fill && !near; ++k) {
                const size_t o = static_cast<size_t>(b[k]) * p.cols;
                near = within_resolution(ld<T>(p.points, o), ld<T>(p.points, o + 1), ld<T>(p.points, o + 2), v[i][0],
                                         v[i][1], v[i][2], p.res_sq);
            }
            if (!near) b[fill++] = rows[i];
        }
    }
    w.cnt[r] = fill;
}

// RANDOM, pass 1: one thread per point flags an insertion into a full bucket (rank in voxel >= max)
__global__ void vx_random_flags_kernel(VoxelParams p, Work w) {
    const unsigned q = tid_global();
    if (q >= p.cap || w.sk[q].pad != 0u) return;
    w.full[w.sseq[q]] = q - segment_begin(q, w.sk) >= p.max_pts ? 1u : 0u;
}

// RANDOM, pass 2 (random_selection_strategy, DefaultVoxelBucket path, voxel_hash_map.h:617-628): the
// first max points fill the slots, every later one overwrites slot (u64(rand) * max) >> 32, and a slot ends
// with its last writer.  Walking the voxel backwards, the first writer met per slot is the last one; the
// walk stops once every slot is claimed, so a dense voxel costs about max * ln(max) draws, not its size.
constexpr uint32_t kFree = 0xffffffffu;
__global__ void vx_random_pick_kernel(VoxelParams p, Work w) {
    const unsigned r = tid_global();
    if (r >= p.cap) return;
    const unsigned nv = w.vrank[p.cap - 1];
    if (r >= nv) {
        w.cnt[r] = 0;
        return;
    }
    const Seg sg = segment_of(r, p.cap, w.sk, w.seg_start);
    uint32_t* b = w.slot + sg.start;
    const unsigned keep = sg.len < p.max_pts ? sg.len : static_cast<unsigned>(p.max_pts);
    if (sg.len > keep) {
        for (unsigned k = 0; k < keep; ++k) b[k] = kFree;
        unsigned claimed = 0;
        for (unsigned k = sg.len; k-- > keep && claimed < keep;) {
            const unsigned q = sg.start + k;
            const uint32_t v = xs_state_after(static_cast<unsigned long long>(w.draw[w.sseq[q]]) + 1ull);
            const unsigned j = static_cast<unsigned>((static_cast<unsigned long long>(v) * p.max_pts) >> 32);
            if (b[j] == kFree) {
                b[j] = row_of(p, w.sseq, q);
                ++claimed;
            }
        }
        for (unsigned k = 0; k < keep; ++k)
            if (b[k] == kFree) b[k] = row_of(p, w.sseq, sg.start + k);
    } else {
        for (unsigned k = 0; k < keep; ++k) b[k] = row_of(p, w.sseq, sg.start + k);
    }
    w.cnt[r] = keep;
}

// ---- 5. emit ----
template <typename T>
__global__ void vx_emit_kernel(VoxelParams p, Work w, const uint32_t* coff, double* out, double* out_n, uint32_t* out_idx,
                               unsigned long long* n_out) {
    const unsigned r = tid_global();
    if (r >= p.cap) return;
    if (r == 0) *n_out = coff[p.cap - 1];
    if (r >= w.vrank[p.cap - 1]) return;
    const unsigned c = w.cnt[r];
    if (c == 0) return;
    const size_t base = coff[r] - c;
    if (p.mode == OB_VOXEL_AVERAGE_POINT || p.mode == OB_VOXEL_POINT_NORMAL) {
        const unsigned cols = p.mode == OB_VOXEL_AVERAGE_POINT ? p.cols : 3u;
        const double* src = w.vres + static_cast<size_t>(r) * (p.mode == OB_VOXEL_AVERAGE_POINT ? p.cols : 6u);
        for (unsigned k = 0; k < cols; ++k) out[base * cols + k] = src[k];
        if (out_n)
            for (unsigned k = 0; k < 3; ++k) out_n[base * 3 + k] = src[3 + k];
        if (out_idx) out_idx[base] = w.vfirst[r];
        return;
    }
    const uint32_t* b = w.slot + w.seg_start[r];
    for (unsigned k = 0; k < c; ++k) {
        const size_t row = b[k];
        for (unsigned m = 0; m < p.cols; ++m) out[(base + k) * p.cols + m] = ld<T>(p.points, row * p.cols + m);
        if (out_idx) out_idx[base + k] = static_cast<uint32_t>(row);
    }
}

}  // namespace

}  // namespace ob

using namespace ob;

namespace {

// the whole pipeline on device buffers; n_out_dev receives the row count
template <typename T>
cudaError_t run_voxel(VoxelParams p, Staging& stg, cudaStream_t st, double* out, double* out_n, uint32_t* out_idx,
                      unsigned long long* n_out_dev) {
    const unsigned cap = p.cap;
    const unsigned nb = blocks_for(cap);
    const int n = static_cast<int>(cap);
    // CUB temporary storage: one block sized for the largest of the calls below
    VKey* k = nullptr;
    uint32_t* u = nullptr;
    CubTemp tmp(stg, sort_pairs(k, k, u, u, n, VKeyDecomposer{}, 0, kKeyBits, st), sort_pairs(u, u, u, u, n, 0, 32, st),
                inclusive_sum(u, u, n, st), exclusive_sum(u, u, n, st));
    if (p.mode == OB_VOXEL_SHUFFLE_FIRST) {
        auto* jkey = stg.scratch<uint32_t>(cap);
        auto* step = stg.scratch<uint32_t>(cap);
        auto* sj = stg.scratch<uint32_t>(cap);
        auto* ss = stg.scratch<uint32_t>(cap);
        auto* where = stg.scratch<uint32_t>(cap);
        auto* order = stg.scratch<uint32_t>(cap);
        auto* last_of = stg.scratch<int32_t>(cap);
        cudaError_t e = stg.error();
        if (e == cudaSuccess) e = cudaMemsetAsync(last_of, 0xff, cap * 4ull, st);
        if (e != cudaSuccess) return e;
        launch(OB_FAM_VOXEL, vx_shuffle_draw_kernel, nb, 256, 0, st, p, jkey, step);
        e = tmp.run(sort_pairs(jkey, sj, step, ss, n, 0, bits_for(cap), st));
        if (e != cudaSuccess) return e;
        launch(OB_FAM_VOXEL, vx_shuffle_index_kernel, nb, 256, 0, st, cap, sj, ss, where, last_of);
        launch(OB_FAM_VOXEL, vx_shuffle_perm_kernel, nb, 256, 0, st, p, sj, ss, where, last_of, order);
        p.order = order;
    }
    auto* keys = stg.scratch<VKey>(cap);
    auto* sk = stg.scratch<VKey>(cap);
    auto* seq = stg.scratch<uint32_t>(cap);
    auto* sseq = stg.scratch<uint32_t>(cap);
    auto* opens = stg.scratch<uint32_t>(cap);
    auto* vrank = stg.scratch<uint32_t>(cap);
    auto* seg_start = stg.scratch<uint32_t>(cap);
    auto* cnt = stg.scratch<uint32_t>(cap);
    auto* coff = stg.scratch<uint32_t>(cap);
    Work w{};
    w.vfirst = stg.scratch<uint32_t>(cap);
    const bool sums = p.mode == OB_VOXEL_AVERAGE_POINT || p.mode == OB_VOXEL_POINT_NORMAL;
    if (sums) w.vres = stg.scratch<double>(static_cast<size_t>(cap) * (p.mode == OB_VOXEL_AVERAGE_POINT ? p.cols : 6u));
    else w.slot = stg.scratch<uint32_t>(cap);
    uint32_t* draw = nullptr;
    if (p.mode == OB_VOXEL_RANDOM) {
        w.full = stg.scratch<uint32_t>(cap);
        draw = stg.scratch<uint32_t>(cap);
    }
    cudaError_t e = stg.error();
    if (e == cudaSuccess && p.mode == OB_VOXEL_RANDOM) e = cudaMemsetAsync(w.full, 0, cap * 4ull, st);
    if (e != cudaSuccess) return e;
    w.sk = sk;
    w.sseq = sseq;
    w.vrank = vrank;
    w.seg_start = seg_start;
    w.cnt = cnt;
    w.draw = draw;
    launch(OB_FAM_VOXEL, vx_key_kernel<T>, nb, 256, 0, st, p, keys, seq);
    e = tmp.run(sort_pairs(keys, sk, seq, sseq, n, VKeyDecomposer{}, 0, kKeyBits, st));
    if (e != cudaSuccess) return e;
    launch(OB_FAM_VOXEL, vx_head_kernel, nb, 256, 0, st, cap, sk, sseq, opens);
    e = tmp.run(inclusive_sum(opens, vrank, n, st));
    if (e != cudaSuccess) return e;
    launch(OB_FAM_VOXEL, vx_seg_kernel, nb, 256, 0, st, cap, sk, sseq, vrank, seg_start);
    if (sums) {
        launch(OB_FAM_VOXEL, vx_reduce_sum_kernel<T>, nb, 256, 0, st, p, w);
    } else if (p.mode == OB_VOXEL_RANDOM) {
        launch(OB_FAM_VOXEL, vx_random_flags_kernel, nb, 256, 0, st, p, w);
        e = tmp.run(exclusive_sum(w.full, draw, n, st));
        if (e != cudaSuccess) return e;
        launch(OB_FAM_VOXEL, vx_random_pick_kernel, nb, 256, 0, st, p, w);
    } else {
        launch(OB_FAM_VOXEL, vx_reduce_first_kernel<T>, nb, 256, 0, st, p, w);
    }
    e = tmp.run(inclusive_sum(cnt, coff, n, st));
    if (e != cudaSuccess) return e;
    launch(OB_FAM_VOXEL, vx_emit_kernel<T>, nb, 256, 0, st, p, w, coff, out, out_n, out_idx, n_out_dev);
    return cudaGetLastError();
}

}  // namespace

extern "C" ob_status ob_voxel_downsample(const ob_voxel_io* io, ob_stream* s) {
    if (!io || !s || !io->n_out) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const int mode = io->mode;
    if (mode < OB_VOXEL_FIRST_N_POINT || mode > OB_VOXEL_POINT_NORMAL) return fail(OB_INVALID_ARGUMENT, "unknown voxel mode");
    if (io->dtype != OB_F32 && io->dtype != OB_F64) return fail(OB_INVALID_ARGUMENT, "unknown dtype");
    // checks in the reference's order (voxel_downsample.cpp:24-32; voxel_hash_map.cpp:317, 355-357, 15-28)
    if (mode == OB_VOXEL_POINT_NORMAL) {
        if (io->cols != 3) return fail(OB_INVALID_ARGUMENT, "voxel_downsample_with_normals expects Nx3 inputs");
        if (!(io->voxel_size > 0.0)) return fail(OB_INVALID_ARGUMENT, "voxel_downsample_with_normals voxel_size must be > 0");
    }
    const size_t cap = row_capacity(io->n, io->n_device, io->capacity);
    if (cap != 0) {  // an empty frame returns before any other check
        if (mode == OB_VOXEL_SHUFFLE_FIRST && io->cols != 3) return fail(OB_INVALID_ARGUMENT, "voxel_downsample: points must be Nx3");
        if (mode != OB_VOXEL_POINT_NORMAL && io->cols < 3)
            return fail(OB_INVALID_ARGUMENT, "voxel_downsample_xd: frame must have at least 3 columns");
        if (mode <= OB_VOXEL_RANDOM) {
            if (io->max_points_per_voxel == 0) return fail(OB_INVALID_ARGUMENT, "max_points_per_voxel must be greater than 0");
            if (io->voxel_size <= 0) return fail(OB_INVALID_ARGUMENT, "voxel_size must be greater than 0");
        }
    }
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    CountedRows res(io->n_out, cap, stg, st, "voxel count");  // outputs hold `cap` rows: never too small
    rs = res.zero();
    if (rs != OB_OK || cap == 0) return rs;
    if (io->cols > 0xffffu) return fail(OB_INVALID_ARGUMENT, "too many points in one call");
    Rows r{};
    rs = count_rows(io->n, io->n_device, io->capacity, &r);
    if (rs != OB_OK) return rs;
    if (!io->points || !io->points_out) return fail(OB_INVALID_ARGUMENT, "null points buffer");
    if (mode == OB_VOXEL_POINT_NORMAL && !io->normals) return fail(OB_INVALID_ARGUMENT, "null normals buffer");
    rs = res.refuse({io->points_out, io->normals_out, io->indices_out}, "a device-side count needs device outputs");
    if (rs != OB_OK) return rs;
    const size_t esz = io->dtype == OB_F64 ? 8 : 4;
    const size_t cols = io->cols, out_cols = mode == OB_VOXEL_POINT_NORMAL ? 3 : cols;
    VoxelParams p{};
    p.points = stg.in(io->points, cap * cols * esz);
    if (mode == OB_VOXEL_POINT_NORMAL) p.normals = stg.in(io->normals, cap * 3 * esz);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage voxel inputs");
    p.n_dev = r.n_dev;
    p.n_host = r.n_host;
    p.cap = r.cap;
    p.cols = static_cast<unsigned>(cols);
    p.mode = mode;
    p.inv = 1.0 / io->voxel_size;  // VoxelHashMap::inv_voxel_size_, voxel_hash_map.cpp:40 / :290
    if (mode == OB_VOXEL_POINT_NORMAL) {
        p.max_pts = 1;
        p.min_pts = 1;
    } else if (mode == OB_VOXEL_SHUFFLE_FIRST) {
        p.max_pts = 1;
        p.min_pts = 1;
        p.res_sq = 0.0;  // nothing to compare against: the first point of a voxel is admitted, the rest are not
    } else {
        p.max_pts = io->max_points_per_voxel;
        p.min_pts = io->min_pts_threshold;
        p.res_sq = io->voxel_size * io->voxel_size / static_cast<double>(io->max_points_per_voxel);  // :39
    }
    double* dpts = res.array(io->points_out, out_cols * 8);
    double* dnrm = mode == OB_VOXEL_POINT_NORMAL ? res.array(io->normals_out, 3 * 8) : nullptr;
    uint32_t* didx = res.array(io->indices_out, 4);
    unsigned long long* dcount = res.word();
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage voxel outputs");
    cudaError_t e = io->dtype == OB_F64 ? run_voxel<double>(p, stg, st, dpts, dnrm, didx, dcount)
                                        : run_voxel<float>(p, stg, st, dpts, dnrm, didx, dcount);
    if (e != cudaSuccess) return fail_cuda(e, "voxel downsample launch");
    return res.finish(dcount);
}
