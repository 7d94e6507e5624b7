// ob_voxel_map.cu -- frame-to-map registration (DESIGN f-6): a device-resident VoxelHashMap3d and
// ICPRegistration::align_points_to_map / build_linear_system.
//
// What it replaces (reference paths relative to the reference tree, ouster-sdk 1.0.1):
//   VoxelHashMap3d (first_n_point, DefaultVoxelBucket)  ouster_core/include/ouster/core/voxel_hash_map.h:287-301, 352-510
//                                                        ouster_core/src/voxel_hash_map.cpp:14-247
//   ICPRegistration, build_linear_system               ouster_mapping/src/icp_registration.cpp
//   Sophus SO3::expAndTheta / leftJacobian, SE3::exp, composition, matrix()
//                                                        thirdparty/sophus/sophus/{so3,se3}.hpp
//   Eigen LDLT (diagonal pivoting) and its solve        jtj.ldlt().solve(-jtr)
//
// The map is an open-addressing hash table in HBM (linear probing, power-of-two capacity).  A slot holds an int32
// voxel key, a state (empty / live / tombstone / being claimed), a 64-bit creation stamp, a fill count and
// max_points_per_voxel double3 points.  Erased voxels become tombstones: queries and inserts probe past them, and
// they are dropped when the table is rebuilt (DESIGN 9).
//
// VoxelHashMapXd (DESIGN f-11) is the same table with num_attributes (A) doubles per point in a separate array of
// cap x max_points_per_voxel x A, allocated only when A > 0: the spatial part stays in the double3 array, so the gate,
// the cull and the searches read exactly what they read for VoxelHashMap3d (A = 0), and only insertion, the rehash,
// emission and the closest-neighbour output touch the attributes.
//
// add_points keys and stable-sorts the batch by voxel (the downsampling pipeline's keys, sort and first-appearance
// numbering, ob_voxel_common.cuh), then one thread per distinct voxel finds or claims its slot and runs the
// first_n_point gate over the voxel's rows in input order, seeded with the points the bucket already holds -- the
// result of inserting the rows one at a time.  A new voxel's stamp is the map's stamp counter plus its
// first-appearance rank in the batch, so voxels are emitted in creation order.
//
// The host keeps an upper bound of the occupied slots (live + tombstones).  Only when that bound plus the batch's
// row capacity could exceed half the table does it read the device counters and the batch's distinct-voxel count
// (one stream synchronisation) and, if needed, rebuild the table for 4 x (live + new voxels) slots, dropping the
// tombstones.  The rebuilt table replaces the old one only after every step succeeded (see reserve()).
//
// align_points_to_map runs its iterations as four kernels each, all on the stream; the convergence flag lives on the
// device and later iterations return at once.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <type_traits>

#include "ob_api_common.h"
#include "ob_cub.cuh"
#include "ob_ldlt.cuh"
#include "ob_rows.cuh"
#include "ob_voxel_common.cuh"

// the slot arrays of the hash table
struct VoxelSlots {
    unsigned cap = 0;          // slots (power of two), 0 before the first insertion
    ob::DeviceBlock key;       // int32 cap x 3
    ob::DeviceBlock state;     // uint32 cap
    ob::DeviceBlock stamp;     // uint64 cap
    ob::DeviceBlock cnt;       // uint32 cap
    ob::DeviceBlock pts;       // double cap x max_pts x 3
    ob::DeviceBlock attr;      // double cap x max_pts x na, empty when na == 0
};

struct ob_voxel_map {
    int device;
    double voxel_size, max_distance, inv, res_sq;
    size_t max_pts, min_pts;
    size_t na;                 // attributes per point (VoxelHashMapXd; 0 for VoxelHashMap3d)
    VoxelSlots slots;
    ob::DeviceBlock ctr;       // device counters, see Ctr
    size_t occupied_bound;     // host upper bound of live + tombstone slots
};

namespace ob {
namespace {

enum : uint32_t { kEmpty = 0, kLive = 1, kTomb = 2, kClaimed = 3 };
// device counters (ob_voxel_map::ctr)
enum { C_STAMP = 0, C_LIVE = 1, C_POINTS = 2, C_OCCUPIED = 3, C_FULL = 4, C_WORDS = 5 };

struct Table {
    unsigned cap;
    int32_t* key;
    uint32_t* state;
    unsigned long long* stamp;
    uint32_t* cnt;
    double* pts;
    unsigned max_pts;
    double* attr;  // max_pts x na per slot, null when na == 0
    unsigned na;
};

Table table_of(const ob_voxel_map* m, const VoxelSlots& s) {
    return Table{s.cap, s.key.get<int32_t>(), s.state.get<uint32_t>(), s.stamp.get<unsigned long long>(),
                 s.cnt.get<uint32_t>(), s.pts.get<double>(), static_cast<unsigned>(m->max_pts), s.attr.get<double>(),
                 static_cast<unsigned>(m->na)};
}
Table table_of(const ob_voxel_map* m) { return table_of(m, m->slots); }
unsigned long long* counters(const ob_voxel_map* m) { return m->ctr.get<unsigned long long>(); }

// columns 0-2 of row `row` of a rows x cols input
template <typename T>
__device__ __forceinline__ void load_xyz(const void* base, size_t row, unsigned cols, double* v) {
    const T* p = static_cast<const T*>(base) + row * cols;
    v[0] = static_cast<double>(p[0]);
    v[1] = static_cast<double>(p[1]);
    v[2] = static_cast<double>(p[2]);
}

__device__ __forceinline__ unsigned slot_hash(int32_t x, int32_t y, int32_t z, unsigned mask) {
    unsigned long long h = static_cast<unsigned long long>(static_cast<uint32_t>(x)) * 0x9E3779B97F4A7C15ull;
    h ^= static_cast<unsigned long long>(static_cast<uint32_t>(y)) * 0xC2B2AE3D27D4EB4Full;
    h ^= static_cast<unsigned long long>(static_cast<uint32_t>(z)) * 0x165667B19E3779F9ull;
    h ^= h >> 32;
    h *= 0xD6E8FEB86659FD93ull;
    h ^= h >> 32;
    return static_cast<unsigned>(h) & mask;
}

__device__ __forceinline__ uint32_t load_state(const uint32_t* s) { return *reinterpret_cast<const volatile uint32_t*>(s); }

// slot of a live voxel, or -1
__device__ __forceinline__ int find_slot(const Table& t, int32_t x, int32_t y, int32_t z) {
    if (t.cap == 0) return -1;
    const unsigned mask = t.cap - 1;
    unsigned i = slot_hash(x, y, z, mask);
    for (unsigned probes = 0; probes < t.cap; ++probes, i = (i + 1) & mask) {
        const uint32_t s = load_state(t.state + i);
        if (s == kEmpty) return -1;
        if (s == kLive && t.key[3 * i] == x && t.key[3 * i + 1] == y && t.key[3 * i + 2] == z) return static_cast<int>(i);
    }
    return -1;
}

// Find the voxel or claim the first empty slot of its probe chain.  Keys are unique inside a batch, so a slot
// another thread claims concurrently never holds this key, and the chain before the first empty slot (all from
// earlier batches) is stable.  Returns the slot; *fresh = 1 for a claimed one (still kClaimed).
__device__ int find_or_claim(const Table& t, int32_t x, int32_t y, int32_t z, unsigned long long* ctr, int* fresh) {
    const unsigned mask = t.cap - 1;
    unsigned i = slot_hash(x, y, z, mask);
    for (unsigned probes = 0; probes < t.cap; ++probes, i = (i + 1) & mask) {
        uint32_t s = load_state(t.state + i);
        if (s == kEmpty) {
            s = atomicCAS(t.state + i, kEmpty, kClaimed);
            if (s == kEmpty) {
                *fresh = 1;
                return static_cast<int>(i);
            }
        }
        if (s == kLive) {
            __threadfence();
            if (t.key[3 * i] == x && t.key[3 * i + 1] == y && t.key[3 * i + 2] == z) {
                *fresh = 0;
                return static_cast<int>(i);
            }
        }
    }
    atomicAdd(ctr + C_FULL, 1ull);  // cannot happen while the host keeps the load at or below one half
    return -1;
}

// ---- add_points ----
template <typename T>
__global__ void vm_key_kernel(Rows r, unsigned cols, double inv, VKey* keys, uint32_t* seq) {
    const unsigned t = tid_global();
    if (t >= r.cap) return;
    VKey k{1u, 0, 0, 0};
    if (t < rows_n(r)) {
        double v[3];
        load_xyz<T>(r.p, t, cols, v);
        k = VKey{0u, floor_cast<int32_t>(mul(v[0], inv)), floor_cast<int32_t>(mul(v[1], inv)),
                 floor_cast<int32_t>(mul(v[2], inv))};
    }
    keys[t] = k;
    seq[t] = t;
}

// one thread per distinct voxel of the batch (first-appearance rank r); rows are cols = 3 + t.na wide, the gate reads
// columns 0-2 and an admitted row's attributes follow it into the slot
template <typename T>
__global__ void vm_insert_kernel(Rows r, unsigned cols, Table t, unsigned long long* ctr, const VKey* sk,
                                 const uint32_t* sseq, const uint32_t* vrank, const uint32_t* seg_start, double res_sq) {
    const unsigned rank = tid_global();
    if (rank >= r.cap || rank >= vrank[r.cap - 1]) return;
    const unsigned start = seg_start[rank];
    const unsigned end = segment_end(start, r.cap, sk);
    const VKey k = sk[start];
    int fresh = 0;
    const int slot = find_or_claim(t, k.x, k.y, k.z, ctr, &fresh);
    if (slot < 0) return;
    if (fresh) {
        t.key[3 * slot] = k.x;
        t.key[3 * slot + 1] = k.y;
        t.key[3 * slot + 2] = k.z;
        t.stamp[slot] = ctr[C_STAMP] + rank;
        t.cnt[slot] = 0;
        __threadfence();
        atomicExch(t.state + slot, kLive);
        atomicAdd(ctr + C_LIVE, 1ull);
        atomicAdd(ctr + C_OCCUPIED, 1ull);
    }
    double* b = t.pts + static_cast<size_t>(slot) * t.max_pts * 3;
    const unsigned before = t.cnt[slot];
    unsigned fill = before;
    for (unsigned q = start; q < end && fill < t.max_pts; ++q) {  // first_n_point, voxel_hash_map.h:287-301
        double v[3];
        load_xyz<T>(r.p, sseq[q], cols, v);
        bool near = false;
        for (unsigned j = 0; j < fill && !near; ++j)
            near = within_resolution(b[3 * j], b[3 * j + 1], b[3 * j + 2], v[0], v[1], v[2], res_sq);
        if (!near) {
            b[3 * fill] = v[0];
            b[3 * fill + 1] = v[1];
            b[3 * fill + 2] = v[2];
            if (t.na) {
                const T* src = static_cast<const T*>(r.p) + static_cast<size_t>(sseq[q]) * cols + 3;
                double* a = t.attr + (static_cast<size_t>(slot) * t.max_pts + fill) * t.na;
                for (unsigned c = 0; c < t.na; ++c) a[c] = static_cast<double>(src[c]);
            }
            ++fill;
        }
    }
    t.cnt[slot] = fill;
    if (fill != before) atomicAdd(ctr + C_POINTS, static_cast<unsigned long long>(fill - before));
}

__global__ void vm_advance_stamp_kernel(unsigned cap, const uint32_t* vrank, unsigned long long* ctr) {
    ctr[C_STAMP] += vrank[cap - 1];
}

// move the live voxels of `o` into the empty table `t`
__global__ void vm_rehash_kernel(Table o, Table t) {
    const unsigned i = tid_global();
    if (i >= o.cap || o.state[i] != kLive) return;
    const int32_t x = o.key[3 * i], y = o.key[3 * i + 1], z = o.key[3 * i + 2];
    const unsigned mask = t.cap - 1;
    unsigned j = slot_hash(x, y, z, mask);
    while (atomicCAS(t.state + j, kEmpty, kClaimed) != kEmpty) j = (j + 1) & mask;
    t.key[3 * j] = x;
    t.key[3 * j + 1] = y;
    t.key[3 * j + 2] = z;
    t.stamp[j] = o.stamp[i];
    t.cnt[j] = o.cnt[i];
    const size_t w = static_cast<size_t>(o.max_pts) * 3;
    for (size_t c = 0; c < static_cast<size_t>(o.cnt[i]) * 3; ++c) t.pts[j * w + c] = o.pts[i * w + c];
    const size_t wa = static_cast<size_t>(o.max_pts) * o.na;
    for (size_t c = 0; c < static_cast<size_t>(o.cnt[i]) * o.na; ++c) t.attr[j * wa + c] = o.attr[i * wa + c];
    t.state[j] = kLive;
}

// ---- remove_voxels_far_from_location (voxel_hash_map.cpp:109-125) ----
// (voxel - origin_voxel).squaredNorm() >= max_voxel_dist_sq in int32 arithmetic, wrapping as x86 does
__global__ void vm_cull_kernel(Table t, unsigned long long* ctr, const double* origin, double inv, int32_t thr,
                               uint32_t* removed) {
    const unsigned i = tid_global();
    if (i >= t.cap) return;
    uint32_t out = 0;
    if (t.state[i] == kLive) {
        const uint32_t ox = static_cast<uint32_t>(floor_cast<int32_t>(mul(origin[0], inv)));
        const uint32_t oy = static_cast<uint32_t>(floor_cast<int32_t>(mul(origin[1], inv)));
        const uint32_t oz = static_cast<uint32_t>(floor_cast<int32_t>(mul(origin[2], inv)));
        const uint32_t dx = static_cast<uint32_t>(t.key[3 * i]) - ox, dy = static_cast<uint32_t>(t.key[3 * i + 1]) - oy,
                       dz = static_cast<uint32_t>(t.key[3 * i + 2]) - oz;
        const int32_t d2 = static_cast<int32_t>((dx * dx + dy * dy) + dz * dz);
        if (d2 >= thr) {
            t.state[i] = kTomb;
            atomicAdd(ctr + C_LIVE, ~0ull);
            atomicAdd(ctr + C_POINTS, 0ull - t.cnt[i]);
            out = 1;
        }
    }
    if (removed) removed[i] = out;
}

// ---- emission in creation order: pointcloud() and the extracted rows ----
__global__ void vm_emit_keys_kernel(Table t, const uint32_t* sel, unsigned long long* keys, uint32_t* slots) {
    const unsigned i = tid_global();
    if (i >= t.cap) return;
    const bool on = sel ? sel[i] != 0 : t.state[i] == kLive;
    keys[i] = on ? t.stamp[i] : ~0ull;
    slots[i] = i;
}
__global__ void vm_emit_counts_kernel(Table t, const unsigned long long* skeys, const uint32_t* sslots, uint32_t* c) {
    const unsigned p = tid_global();
    if (p >= t.cap) return;
    c[p] = skeys[p] != ~0ull ? t.cnt[sslots[p]] : 0u;
}
__global__ void vm_emit_kernel(Table t, const unsigned long long* skeys, const uint32_t* sslots, const uint32_t* off,
                               double* out, unsigned long long capacity, unsigned long long* n_out) {
    const unsigned p = tid_global();
    if (p >= t.cap) return;
    if (p == t.cap - 1) *n_out = off[p];
    if (skeys[p] == ~0ull) return;
    const unsigned s = sslots[p];
    const unsigned c = t.cnt[s];
    const unsigned long long base = off[p] - c;
    const double* b = t.pts + static_cast<size_t>(s) * t.max_pts * 3;
    const double* a = t.attr + static_cast<size_t>(s) * t.max_pts * t.na;
    const unsigned cols = 3 + t.na;
    for (unsigned k = 0; k < c && base + k < capacity; ++k) {
        for (int d = 0; d < 3; ++d) out[(base + k) * cols + d] = b[3 * k + d];
        for (unsigned d = 0; d < t.na; ++d) out[(base + k) * cols + 3 + d] = a[k * t.na + d];
    }
}

// ---- get_closest_neighbor (voxel_hash_map.cpp:194-247) ----
__constant__ int8_t kShift[27][3] = {
    {0, 0, 0},   {1, 0, 0},   {-1, 0, 0},  {0, 1, 0},   {0, -1, 0},   {0, 0, 1},  {0, 0, -1},  {1, 1, 0},   {1, -1, 0},
    {-1, 1, 0},  {-1, -1, 0}, {1, 0, 1},   {1, 0, -1},  {-1, 0, 1},   {-1, 0, -1}, {0, 1, 1},  {0, 1, -1},  {0, -1, 1},
    {0, -1, -1}, {1, 1, 1},   {1, 1, -1},  {1, -1, 1},  {1, -1, -1},  {-1, 1, 1}, {-1, 1, -1}, {-1, -1, 1}, {-1, -1, -1},
};

// nearest point to q with squared distance < max_d2, visiting the 27 voxels in VOXEL_SHIFTS order and pruning each by
// its AABB lower bound; (0,0,0) and max_d2 when nothing qualifies.  kAt: *at = the point's index in the attribute
// array (slot * max_pts + k), or -1
template <bool kAt = false>
__device__ double closest(const Table& t, double inv, double vs, const double* q, double max_d2, double* nb,
                          long long* at = nullptr) {
    const int32_t v[3] = {floor_cast<int32_t>(mul(q[0], inv)), floor_cast<int32_t>(mul(q[1], inv)),
                          floor_cast<int32_t>(mul(q[2], inv))};
    double best = max_d2;
    nb[0] = nb[1] = nb[2] = 0.0;
    if (kAt) *at = -1;
    for (int s = 0; s < 27; ++s) {
        int32_t w[3];
        double lb = 0.0;
        for (int d = 0; d < 3; ++d) {
            w[d] = static_cast<int32_t>(static_cast<uint32_t>(v[d]) + static_cast<uint32_t>(kShift[s][d]));
            const double lo = mul(static_cast<double>(w[d]), vs);
            const double hi = add(lo, vs);
            if (q[d] < lo) {
                const double delta = sub(lo, q[d]);
                lb = add(lb, mul(delta, delta));
            } else if (q[d] > hi) {
                const double delta = sub(q[d], hi);
                lb = add(lb, mul(delta, delta));
            }
        }
        if (lb >= best) continue;
        const int slot = find_slot(t, w[0], w[1], w[2]);
        if (slot < 0) continue;
        const double* b = t.pts + static_cast<size_t>(slot) * t.max_pts * 3;
        const unsigned c = t.cnt[slot];
        for (unsigned k = 0; k < c; ++k) {
            const double d2 = sqn3(sub(b[3 * k], q[0]), sub(b[3 * k + 1], q[1]), sub(b[3 * k + 2], q[2]));
            if (d2 < best) {
                best = d2;
                nb[0] = b[3 * k];
                nb[1] = b[3 * k + 1];
                nb[2] = b[3 * k + 2];
                if (kAt) *at = static_cast<long long>(slot) * t.max_pts + k;
            }
        }
    }
    return best;
}

// kAttr: the map has attributes, a neighbour row is 3 + t.na wide (zeros when nothing qualifies,
// PointDefaultValue::make(point_cols())); without, the search does not track where the neighbour lives
template <typename T, bool kAttr>
__global__ void vm_closest_kernel(Rows r, Table t, double inv, double vs, double max_d2, double* nb, double* d2) {
    const unsigned i = tid_global();
    if (i >= r.cap || i >= rows_n(r)) return;
    double q[3], p[3];
    load3<T>(r.p, i, q);
    long long at = -1;
    const double best = closest<kAttr>(t, inv, vs, q, max_d2, p, &at);
    const unsigned cols = kAttr ? 3 + t.na : 3;
    double* o = nb + static_cast<size_t>(i) * cols;
    o[0] = p[0];
    o[1] = p[1];
    o[2] = p[2];
    if (kAttr)
        for (unsigned d = 0; d < t.na; ++d) o[3 + d] = at >= 0 ? t.attr[static_cast<size_t>(at) * t.na + d] : 0.0;
    if (d2) d2[i] = best;
}

// ---- build_linear_system in parallel_deterministic_reduce's tree (icp_registration.cpp) ----
// blocked_range(begin, end, 128) splits at mid = b + (e - b) / 2 while it holds more than 128 pairs; a leaf sums
// its pairs sequentially from zero; a parent is left + right.  Only the 15 entries of the lower triangle of JtJ
// that a pair touches and the 6 of Jtr are stored: every other entry is +0.0 + +0.0 at every node.
constexpr unsigned kGrain = 128;
constexpr int kSys = 21;
// JtJ (row, col) of the stored entries 0..14; Jtr is 15..20
__constant__ uint8_t kJtjRC[15][2] = {{0, 0}, {1, 1}, {2, 2}, {3, 1}, {3, 2}, {4, 0}, {4, 2}, {5, 0},
                                      {5, 1}, {3, 3}, {4, 3}, {4, 4}, {5, 3}, {5, 4}, {5, 5}};

__host__ __device__ inline unsigned tree_depth(unsigned long long n) {
    unsigned d = 0;
    while (n > kGrain) {
        n = (n + 1) / 2;
        ++d;
    }
    return d;
}
// range of node (k, i) (i's k bits, most significant first, choose the child); false when an ancestor is a leaf
__device__ inline bool tree_node(unsigned long long n, unsigned k, unsigned i, unsigned long long* b, unsigned long long* e) {
    unsigned long long lo = 0, hi = n;
    for (unsigned l = 0; l < k; ++l) {
        if (hi - lo <= kGrain) return false;
        const unsigned long long mid = lo + (hi - lo) / 2;
        if ((i >> (k - 1 - l)) & 1u) lo = mid;
        else hi = mid;
    }
    *b = lo;
    *e = hi;
    return true;
}

// the leaf body: pairs [b, e) summed from zero in order
__device__ void leaf_sum(const double* src, const double* tgt, unsigned long long b, unsigned long long e, double ks,
                         double* acc) {
    for (int j = 0; j < kSys; ++j) acc[j] = 0.0;
    const double k2 = mul(ks, ks);
    for (unsigned long long i = b; i < e; ++i) {
        const double sx = src[3 * i], sy = src[3 * i + 1], sz = src[3 * i + 2];
        const double rx = sub(sx, tgt[3 * i]), ry = sub(sy, tgt[3 * i + 1]), rz = sub(sz, tgt[3 * i + 2]);
        const double kr = add(ks, sqn3(rx, ry, rz));
        const double w = k2 / mul(kr, kr);
        const double wsx = mul(w, sx), wsy = mul(w, sy), wsz = mul(w, sz);
        acc[0] = add(acc[0], w);
        acc[1] = add(acc[1], w);
        acc[2] = add(acc[2], w);
        acc[3] = sub(acc[3], wsz);
        acc[4] = add(acc[4], wsy);
        acc[5] = add(acc[5], wsz);
        acc[6] = sub(acc[6], wsx);
        acc[7] = sub(acc[7], wsy);
        acc[8] = add(acc[8], wsx);
        const double wsx2 = mul(wsx, sx), wsy2 = mul(wsy, sy), wsz2 = mul(wsz, sz);
        acc[9] = add(acc[9], add(wsy2, wsz2));
        acc[10] = sub(acc[10], mul(wsx, sy));
        acc[11] = add(acc[11], add(wsx2, wsz2));
        acc[12] = sub(acc[12], mul(wsx, sz));
        acc[13] = sub(acc[13], mul(wsy, sz));
        acc[14] = add(acc[14], add(wsx2, wsy2));
        acc[15] = add(acc[15], mul(w, rx));
        acc[16] = add(acc[16], mul(w, ry));
        acc[17] = add(acc[17], mul(w, rz));
        const double cx = sub(mul(sy, rz), mul(sz, ry)), cy = sub(mul(sz, rx), mul(sx, rz)), cz = sub(mul(sx, ry), mul(sy, rx));
        acc[18] = add(acc[18], mul(w, cx));
        acc[19] = add(acc[19], mul(w, cy));
        acc[20] = add(acc[20], mul(w, cz));
    }
}

// one thread per slot of the deepest level; the thread whose path ends at a leaf with all remaining bits zero owns it
__global__ void icp_leaf_kernel(const double* src, const double* tgt, const unsigned long long* n_pairs,
                                unsigned long long max_n, double ks, const int* done, unsigned slots, double* val) {
    if (done && *done) return;
    const unsigned t = tid_global();
    const unsigned long long n = n_pairs ? min(*n_pairs, max_n) : max_n;
    const unsigned D = tree_depth(n);
    if (t >= slots || t >= (1u << D)) return;
    unsigned long long lo = 0, hi = n;
    unsigned l = 0;
    for (; l < D && hi - lo > kGrain; ++l) {
        const unsigned long long mid = lo + (hi - lo) / 2;
        if ((t >> (D - 1 - l)) & 1u) lo = mid;
        else hi = mid;
    }
    if (t & ((1u << (D - l)) - 1u)) return;
    double acc[kSys];
    leaf_sum(src, tgt, lo, hi, ks, acc);
    for (int j = 0; j < kSys; ++j) val[static_cast<size_t>(t) * kSys + j] = acc[j];
}

// parents bottom-up (one block): node (k, i) lives in slot i << (D - k), its right child in (2i + 1) << (D - k - 1)
__device__ void tree_reduce(unsigned long long n, double* val) {
    const unsigned D = tree_depth(n);
    for (int k = static_cast<int>(D) - 1; k >= 0; --k) {
        for (unsigned i = threadIdx.x; i < (1u << k); i += blockDim.x) {
            unsigned long long b, e;
            if (!tree_node(n, static_cast<unsigned>(k), i, &b, &e) || e - b <= kGrain) continue;
            double* l = val + (static_cast<size_t>(i) << (D - k)) * kSys;
            const double* r = val + (static_cast<size_t>(2 * i + 1) << (D - k - 1)) * kSys;
            for (int j = 0; j < kSys; ++j) l[j] = add(l[j], r[j]);
        }
        __syncthreads();
    }
}

// unpack the root: JtJ (6x6 row-major, lower triangle; the rest +0.0) and Jtr
__device__ void unpack_system(const double* v, double* jtj, double* jtr) {
    for (int j = 0; j < 36; ++j) jtj[j] = 0.0;
    for (int j = 0; j < 15; ++j) jtj[kJtjRC[j][0] * 6 + kJtjRC[j][1]] = v[j];
    for (int j = 0; j < 6; ++j) jtr[j] = v[15 + j];
}

// ---- Sophus (quaternion x, y, z, w; translation) ----
struct SE3 {
    double q[4];  // x, y, z, w
    double t[3];
};

__device__ void cross3(const double* a, const double* b, double* c) {
    c[0] = sub(mul(a[1], b[2]), mul(a[2], b[1]));
    c[1] = sub(mul(a[2], b[0]), mul(a[0], b[2]));
    c[2] = sub(mul(a[0], b[1]), mul(a[1], b[0]));
}
// SO3 * p (so3.hpp:388-397): uv = q.vec() x p; uv += uv; p + w * uv + q.vec() x uv
__device__ void rotate(const double* q, const double* p, double* out) {
    double uv[3], c[3];
    cross3(q, p, uv);
    for (int d = 0; d < 3; ++d) uv[d] = add(uv[d], uv[d]);
    cross3(q, uv, c);
    for (int d = 0; d < 3; ++d) out[d] = add(add(p[d], mul(q[3], uv[d])), c[d]);
}
// SE3 * p (se3.hpp:319-322)
__device__ void se3_apply(const SE3& g, const double* p, double* out) {
    double r[3];
    rotate(g.q, p, r);
    for (int d = 0; d < 3; ++d) out[d] = add(r[d], g.t[d]);
}
// a * b (se3.hpp:302-306, so3.hpp:344-369 with SO3's normalising constructor, so3.hpp:527-534)
__device__ SE3 se3_mul(const SE3& a, const SE3& b) {
    SE3 c;
    const double ax = a.q[0], ay = a.q[1], az = a.q[2], aw = a.q[3];
    const double bx = b.q[0], by = b.q[1], bz = b.q[2], bw = b.q[3];
    c.q[3] = sub(sub(sub(mul(aw, bw), mul(ax, bx)), mul(ay, by)), mul(az, bz));
    c.q[0] = sub(add(add(mul(aw, bx), mul(ax, bw)), mul(ay, bz)), mul(az, by));
    c.q[1] = sub(add(add(mul(aw, by), mul(ay, bw)), mul(az, bx)), mul(ax, bz));
    c.q[2] = sub(add(add(mul(aw, bz), mul(az, bw)), mul(ax, by)), mul(ay, bx));
    // coeffs() (x, y, z, w).norm() as Eigen's two-lane reduction sums it
    const double len = sqrt(add(add(mul(c.q[0], c.q[0]), mul(c.q[2], c.q[2])), add(mul(c.q[1], c.q[1]), mul(c.q[3], c.q[3]))));
    for (int j = 0; j < 4; ++j) c.q[j] = c.q[j] / len;
    double r[3];
    rotate(a.q, b.t, r);
    for (int d = 0; d < 3; ++d) c.t[d] = add(a.t[d], r[d]);
    return c;
}
// SE3::exp (se3.hpp:852-861): SO3::expAndTheta (so3.hpp:694-731), SO3::leftJacobian(omega, theta) (so3.hpp:550-571)
__device__ SE3 se3_exp(const double* a) {
    const double eps = DBL_EPSILON;
    const double* om = a + 3;
    const double theta_sq = sqn3(om[0], om[1], om[2]);
    double theta, imag, real;
    if (theta_sq < mul(eps, eps)) {
        theta = 0.0;
        const double po4 = mul(theta_sq, theta_sq);
        imag = add(sub(0.5, mul(1.0 / 48.0, theta_sq)), mul(1.0 / 3840.0, po4));
        real = add(sub(1.0, mul(1.0 / 8.0, theta_sq)), mul(1.0 / 384.0, po4));
    } else {
        theta = sqrt(theta_sq);
        const double half = mul(0.5, theta);
        imag = sin(half) / theta;
        real = cos(half);
    }
    SE3 g;
    g.q[0] = mul(imag, om[0]);
    g.q[1] = mul(imag, om[1]);
    g.q[2] = mul(imag, om[2]);
    g.q[3] = real;
    const double O[3][3] = {{0.0, -om[2], om[1]}, {om[2], 0.0, -om[0]}, {-om[1], om[0], 0.0}};
    double V[3][3];
    const double tsq = mul(theta, theta);
    if (tsq < mul(eps, eps)) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) V[i][j] = add(i == j ? 1.0 : 0.0, mul(0.5, O[i][j]));
    } else {
        const double c1 = sub(1.0, cos(theta)) / tsq;
        const double c2 = sub(theta, sin(theta)) / mul(tsq, theta);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                const double o2 = add(add(mul(O[i][0], O[0][j]), mul(O[i][1], O[1][j])), mul(O[i][2], O[2][j]));
                V[i][j] = add(add(i == j ? 1.0 : 0.0, mul(c1, O[i][j])), mul(c2, o2));
            }
    }
    for (int i = 0; i < 3; ++i) g.t[i] = add(add(mul(V[i][0], a[0]), mul(V[i][1], a[1])), mul(V[i][2], a[2]));
    return g;
}
// SE3::matrix() (se3.hpp:273-289; Eigen Quaternion::toRotationMatrix), row-major 4x4
__device__ void se3_matrix(const SE3& g, double* M) {
    const double x = g.q[0], y = g.q[1], z = g.q[2], w = g.q[3];
    const double tx = mul(2.0, x), ty = mul(2.0, y), tz = mul(2.0, z);
    const double twx = mul(tx, w), twy = mul(ty, w), twz = mul(tz, w);
    const double txx = mul(tx, x), txy = mul(ty, x), txz = mul(tz, x);
    const double tyy = mul(ty, y), tyz = mul(tz, y), tzz = mul(tz, z);
    const double R[9] = {sub(1.0, add(tyy, tzz)), sub(txy, twz),           add(txz, twy),
                         add(txy, twz),           sub(1.0, add(txx, tzz)), sub(tyz, twx),
                         sub(txz, twy),           add(tyz, twx),           sub(1.0, add(txx, tyy))};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) M[i * 4 + j] = R[i * 3 + j];
        M[i * 4 + 3] = g.t[i];
    }
    M[12] = M[13] = M[14] = 0.0;
    M[15] = 1.0;
}

// ---- align_points_to_map (icp_registration.cpp) ----
struct IcpState {
    SE3 inc;         // the previous iteration's estimation, applied to the source by the next association
    SE3 pose;        // t_icp
    int has_inc;
    int done;        // converged, or the map is empty
    int iterations;
    int pad;
    unsigned long long n_pairs;
};

constexpr unsigned kAssocThreads = 256;

template <typename T>
__global__ void icp_init_kernel(Rows r, const unsigned long long* ctr, double* src, IcpState* s) {
    const unsigned i = tid_global();
    if (i == 0) {
        IcpState z{};
        z.pose.q[3] = 1.0;
        z.inc.q[3] = 1.0;
        z.done = ctr[C_LIVE] == 0 ? 1 : 0;  // an empty map returns the identity
        *s = z;
    }
    if (i >= r.cap || i >= rows_n(r)) return;
    load3<T>(r.p, i, src + 3 * i);
}

// association (icp_registration.cpp data_association), fused with applying the previous increment in place
__global__ void icp_assoc_kernel(Rows r, Table t, double inv, double vs, double max_d2, double* src, double* tgt,
                                 uint32_t* valid, uint32_t* block_count, IcpState* s) {
    if (s->done) return;
    const unsigned i = tid_global();
    const unsigned n = rows_n(r);
    bool ok = false;
    if (i < n) {
        double p[3] = {src[3 * i], src[3 * i + 1], src[3 * i + 2]};
        if (s->has_inc) {
            double q[3];
            se3_apply(s->inc, p, q);
            for (int d = 0; d < 3; ++d) src[3 * i + d] = p[d] = q[d];
        }
        double nb[3];
        const double d2 = closest(t, inv, vs, p, max_d2, nb);
        ok = d2 < max_d2;
        if (ok)
            for (int d = 0; d < 3; ++d) tgt[3 * i + d] = nb[d];
    }
    if (i < r.cap) valid[i] = ok ? 1u : 0u;
    const int c = __syncthreads_count(ok);
    if (threadIdx.x == 0) block_count[blockIdx.x] = static_cast<uint32_t>(c);
}

// order-preserving compaction of the valid pairs; the last block writes the pair count
__global__ void icp_compact_kernel(unsigned cap, const double* src, const double* tgt, const uint32_t* valid,
                                   const uint32_t* block_count, double* ps, double* pt, IcpState* s) {
    if (s->done) return;
    compact_rows<kAssocThreads>(cap, valid, block_count, &s->n_pairs, [&](unsigned i, size_t o) {
        for (int d = 0; d < 3; ++d) {
            ps[3 * o + d] = src[3 * static_cast<size_t>(i) + d];
            pt[3 * o + d] = tgt[3 * static_cast<size_t>(i) + d];
        }
    });
}

// the tree's parents, then (thread 0) the LDLT solve, SE3::exp, t_icp = estimation * t_icp and the stop test
constexpr unsigned kTreeThreads = 256;

__global__ void __launch_bounds__(kTreeThreads, 1) icp_solve_kernel(double* val, double crit_sq, IcpState* s) {
    if (s->done) return;
    const unsigned long long n = s->n_pairs;
    tree_reduce(n, val);
    if (threadIdx.x != 0) return;
    double jtj[36], jtr[6], rhs[6], dx[6];
    unpack_system(val, jtj, jtr);
    for (int j = 0; j < 6; ++j) rhs[j] = -jtr[j];
    ldlt_solve6(jtj, rhs, dx);
    const SE3 est = se3_exp(dx);
    s->pose = se3_mul(est, s->pose);
    s->inc = est;
    s->has_inc = 1;
    s->iterations += 1;
    // Vector6d::squaredNorm in Eigen's two-lane order
    const double l0 = add(mul(dx[0], dx[0]), add(mul(dx[2], dx[2]), mul(dx[4], dx[4])));
    const double l1 = add(mul(dx[1], dx[1]), add(mul(dx[3], dx[3]), mul(dx[5], dx[5])));
    if (add(l0, l1) < crit_sq) s->done = 1;
}

__global__ void icp_finish_kernel(const IcpState* s, double* pose, int32_t* iterations) {
    se3_matrix(s->pose, pose);
    if (iterations) *iterations = s->iterations;
}

// build_linear_system on its own: the root of the tree, unpacked
__global__ void __launch_bounds__(kTreeThreads, 1) icp_system_kernel(const unsigned long long* n_pairs,
                                                                    unsigned long long max_n, double* val, double* jtj,
                                                                    double* jtr) {
    const unsigned long long n = n_pairs ? min(*n_pairs, max_n) : max_n;
    tree_reduce(n, val);
    if (threadIdx.x == 0) unpack_system(val, jtj, jtr);
}

}  // namespace
}  // namespace ob

using namespace ob;

namespace {

size_t table_bytes(size_t cap, size_t max_pts, size_t na) { return cap * (12 + 4 + 8 + 4 + (24 + 8 * na) * max_pts); }

// a new, empty table of `cap` slots for the map `m` in `t`
cudaError_t alloc_table(const ob_voxel_map* m, unsigned cap, cudaStream_t st, VoxelSlots* t) {
    t->cap = cap;
    cudaError_t e = t->key.alloc(cap * 12ull);
    if (e == cudaSuccess) e = t->state.alloc(cap * 4ull);
    if (e == cudaSuccess) e = t->stamp.alloc(cap * 8ull);
    if (e == cudaSuccess) e = t->cnt.alloc(cap * 4ull);
    if (e == cudaSuccess) e = t->pts.alloc(cap * m->max_pts * 24ull);
    if (e == cudaSuccess && m->na) e = t->attr.alloc(cap * m->max_pts * m->na * 8ull);
    if (e == cudaSuccess) e = cudaMemsetAsync(t->state.get(), 0, cap * 4ull, st);
    return e;
}

constexpr unsigned kMinSlots = 1024;

// Make room before a batch of at most `rows` rows whose distinct voxel count is the device word *nv_dev (the batch
// is already sorted and numbered).  The map waits for the host only here, and only when the host bound of occupied
// slots plus `rows` could pass half the table: then it reads the counters and nv, and grows to the next power of two
// >= 4 (live + nv) slots if live + tombstones + nv would pass half.  The new table is built and filled on the side
// and committed only when every step succeeded; any failure leaves the map as it was.  *added = what the batch can
// add to the occupied slots (rows, or the exact nv once it was read).
ob_status reserve(ob_voxel_map* m, size_t rows, const uint32_t* nv_dev, cudaStream_t st, size_t* added) {
    *added = rows;
    if (m->slots.cap && m->occupied_bound + rows <= m->slots.cap / 2) return OB_OK;
    unsigned long long c[C_WORDS] = {};
    uint32_t nv = 0;
    cudaError_t e = cudaMemcpyAsync(c, counters(m), sizeof(c), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&nv, nv_dev, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map counters");
    *added = nv;
    m->occupied_bound = static_cast<size_t>(c[C_OCCUPIED]);
    if (m->slots.cap && m->occupied_bound + nv <= m->slots.cap / 2) return OB_OK;
    const size_t live = static_cast<size_t>(c[C_LIVE]);
    const size_t need = 4 * (live + nv);
    size_t cap = kMinSlots;
    while (cap < need) cap <<= 1;
    size_t free_b = 0, total_b = 0;
    e = cudaMemGetInfo(&free_b, &total_b);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map allocation");
    if (cap > (1ull << 31) || table_bytes(cap, m->max_pts, m->na) > free_b)
        return fail(OB_RUNTIME_ERROR, "voxel map: a table of " + std::to_string(cap) + " slots (" +
                                          std::to_string(table_bytes(cap, m->max_pts, m->na)) +
                                          " bytes) does not fit in free device memory");
    VoxelSlots nt;
    e = alloc_table(m, static_cast<unsigned>(cap), st, &nt);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map allocation");
    if (m->slots.cap) {
        launch(OB_FAM_VOXEL_MAP, vm_rehash_kernel, blocks_for(m->slots.cap), 256, 0, st, table_of(m), table_of(m, nt));
        e = cudaGetLastError();
    }
    const unsigned long long occ = live;
    if (e == cudaSuccess) e = cudaMemcpyAsync(counters(m) + C_OCCUPIED, &occ, 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // the old table is freed below, `occ` is on this stack
    if (e != cudaSuccess) return fail_cuda(e, "voxel map rehash");
    m->slots = std::move(nt);
    m->occupied_bound = live;
    return OB_OK;
}

// a batch keyed, sorted and numbered by voxel (the first half of add_points)
struct AddBatch {
    VKey* sk;
    uint32_t *sseq, *vrank, *seg_start;
};

template <typename T>
cudaError_t sort_batch(const ob_voxel_map* m, Rows r, unsigned cols, Staging& stg, cudaStream_t st, AddBatch* b) {
    const unsigned cap = r.cap;
    const unsigned nb = blocks_for(cap);
    auto* keys = stg.scratch<VKey>(cap);
    b->sk = stg.scratch<VKey>(cap);
    auto* seq = stg.scratch<uint32_t>(cap);
    b->sseq = stg.scratch<uint32_t>(cap);
    auto* opens = stg.scratch<uint32_t>(cap);
    b->vrank = stg.scratch<uint32_t>(cap);
    b->seg_start = stg.scratch<uint32_t>(cap);
    const auto sort = sort_pairs(keys, b->sk, seq, b->sseq, static_cast<int>(cap), VKeyDecomposer{}, 0, kKeyBits, st);
    const auto scan = inclusive_sum(opens, b->vrank, static_cast<int>(cap), st);
    CubTemp tmp(stg, sort, scan);
    if (cudaError_t e = stg.error()) return e;
    launch(OB_FAM_VOXEL_MAP, vm_key_kernel<T>, nb, 256, 0, st, r, cols, m->inv, keys, seq);
    if (cudaError_t e = tmp.run(sort)) return e;
    launch(OB_FAM_VOXEL_MAP, vx_head_kernel, nb, 256, 0, st, cap, b->sk, b->sseq, opens);
    if (cudaError_t e = tmp.run(scan)) return e;
    launch(OB_FAM_VOXEL_MAP, vx_seg_kernel, nb, 256, 0, st, cap, b->sk, b->sseq, b->vrank, b->seg_start);
    return cudaGetLastError();
}

// the second half: every distinct voxel of the batch into the table
template <typename T>
cudaError_t insert_batch(ob_voxel_map* m, Rows r, unsigned cols, const AddBatch& b, cudaStream_t st) {
    launch(OB_FAM_VOXEL_MAP, vm_insert_kernel<T>, blocks_for(r.cap), 256, 0, st, r, cols, table_of(m), counters(m),
           b.sk, b.sseq, b.vrank, b.seg_start, m->res_sq);
    launch(OB_FAM_VOXEL_MAP, vm_advance_stamp_kernel, 1, 1, 0, st, r.cap, b.vrank, counters(m));
    return cudaGetLastError();
}

// rows of the selected voxels (sel == null: every live voxel) in creation order into out (capacity rows);
// *n_dev = the number of rows selected
cudaError_t run_emit(const ob_voxel_map* m, const uint32_t* sel, Staging& stg, cudaStream_t st, double* out,
                     size_t capacity, unsigned long long* n_dev) {
    const unsigned cap = m->slots.cap;
    if (cap == 0) return cudaMemsetAsync(n_dev, 0, 8, st);
    auto* keys = stg.scratch<unsigned long long>(cap);
    auto* skeys = stg.scratch<unsigned long long>(cap);
    auto* slots = stg.scratch<uint32_t>(cap);
    auto* sslots = stg.scratch<uint32_t>(cap);
    auto* c = stg.scratch<uint32_t>(cap);
    auto* off = stg.scratch<uint32_t>(cap);
    const auto sort = sort_pairs(keys, skeys, slots, sslots, static_cast<int>(cap), 0, 64, st);
    const auto scan = inclusive_sum(c, off, static_cast<int>(cap), st);
    CubTemp tmp(stg, sort, scan);
    if (cudaError_t e = stg.error()) return e;
    const Table t = table_of(m);
    const unsigned nb = blocks_for(cap);
    launch(OB_FAM_VOXEL_MAP, vm_emit_keys_kernel, nb, 256, 0, st, t, sel, keys, slots);
    if (cudaError_t e = tmp.run(sort)) return e;
    launch(OB_FAM_VOXEL_MAP, vm_emit_counts_kernel, nb, 256, 0, st, t, skeys, sslots, c);
    if (cudaError_t e = tmp.run(scan)) return e;
    launch(OB_FAM_VOXEL_MAP, vm_emit_kernel, nb, 256, 0, st, t, skeys, sslots, off, out, capacity, n_dev);
    return cudaGetLastError();
}

// rows of the selected voxels of a non-empty map into `out` (null: count only), the count through `res`
ob_status emit_rows(const ob_voxel_map* m, const uint32_t* sel, Staging& stg, cudaStream_t st, double* out,
                    size_t capacity, CountedRows& res, const char* what) {
    double* dout = res.array(out, (3 + m->na) * 8);
    unsigned long long* dn = res.word();
    cudaError_t e = stg.error();
    if (e == cudaSuccess) e = run_emit(m, sel, stg, st, dout, out ? capacity : 0, dn);
    if (e != cudaSuccess) return fail_cuda(e, what);
    return res.finish(dn);
}

const char* const kMixedCount = "a device-side count needs device outputs";

// max_voxel_dist_sq of remove_voxels_far_from_location (voxel_hash_map.cpp:112-113) in x86 int32 arithmetic
int32_t cull_threshold(double max_distance, double inv) {
    const double c = std::ceil(max_distance * inv);
    const uint32_t d = static_cast<uint32_t>(c >= -2147483648.0 && c < 2147483648.0 ? static_cast<int32_t>(c) : INT32_MIN) + 1u;
    return static_cast<int32_t>(d * d);
}

// leaf values of the deterministic-reduce tree for up to `cap` pairs
unsigned tree_slots(size_t cap) { return 1u << tree_depth(cap); }

// sort, make room, insert: the body of ob_voxel_map_add_points / _add_rows for staged rows of `cols` columns
ob_status add_batch(ob_voxel_map* m, Rows r, unsigned cols, bool f64, Staging& stg, cudaStream_t st) {
    AddBatch b{};
    cudaError_t e = f64 ? sort_batch<double>(m, r, cols, stg, st, &b) : sort_batch<float>(m, r, cols, stg, st, &b);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map add_points");
    size_t added = 0;
    ob_status rs = reserve(m, r.cap, b.vrank + r.cap - 1, st, &added);
    if (rs != OB_OK) return rs;  // nothing inserted; the map is as it was
    e = f64 ? insert_batch<double>(m, r, cols, b, st) : insert_batch<float>(m, r, cols, b, st);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map add_points");
    m->occupied_bound += added;
    return OB_OK;
}

const char* const kDimensionError = "VoxelHashMap::add_points received unexpected point dimension";

}  // namespace

extern "C" {

ob_status ob_voxel_map_create(double voxel_size, double max_distance, size_t max_points_per_voxel,
                              size_t min_pts_threshold, int device, ob_voxel_map** out) {
    return ob_voxel_map_create_xd(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold, 0, device, out);
}

ob_status ob_voxel_map_create_xd(double voxel_size, double max_distance, size_t max_points_per_voxel,
                                 size_t min_pts_threshold, size_t num_attributes, int device, ob_voxel_map** out) {
    if (!out) return fail(OB_INVALID_ARGUMENT, "null output pointer");
    // the constructor's checks in its order (voxel_hash_map.cpp:23-31)
    if (max_points_per_voxel == 0) return fail(OB_INVALID_ARGUMENT, "max_points_per_voxel must be greater than 0");
    if (voxel_size <= 0) return fail(OB_INVALID_ARGUMENT, "voxel_size must be greater than 0");
    if (max_distance <= 0) return fail(OB_INVALID_ARGUMENT, "max_distance must be greater than 0");
    if (max_points_per_voxel > 0xffffu) return fail(OB_INVALID_ARGUMENT, "max_points_per_voxel too large");
    if (num_attributes > 0xffffu) return fail(OB_INVALID_ARGUMENT, "num_attributes too large");
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    std::unique_ptr<ob_voxel_map> m(new ob_voxel_map{});
    m->device = device;
    m->voxel_size = voxel_size;
    m->max_distance = max_distance;
    m->max_pts = max_points_per_voxel;
    m->min_pts = min_pts_threshold;
    m->na = num_attributes;
    m->res_sq = voxel_size * voxel_size / static_cast<double>(max_points_per_voxel);  // :38
    m->inv = 1.0 / voxel_size;                                                          // :39
    cudaError_t e = m->ctr.alloc(C_WORDS * 8);
    if (e == cudaSuccess) e = cudaMemset(m->ctr.get(), 0, C_WORDS * 8);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map allocation");
    *out = m.release();
    return OB_OK;
}

ob_status ob_voxel_map_destroy(ob_voxel_map* m) {
    if (!m) return OB_OK;
    DeviceScope on(m->device);
    delete m;
    return OB_OK;
}

ob_status ob_voxel_map_clear(ob_voxel_map* m, ob_stream* s) {
    if (!m || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    cudaError_t e = cudaSuccess;
    if (m->slots.cap) e = cudaMemsetAsync(m->slots.state.get(), 0, m->slots.cap * 4ull, st);
    // the stamp counter keeps running: creation order stays monotone across clears
    if (e == cudaSuccess) e = cudaMemsetAsync(counters(m) + C_LIVE, 0, (C_WORDS - C_LIVE) * 8, st);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map clear");
    m->occupied_bound = 0;
    return OB_OK;
}

ob_status ob_voxel_map_cols(const ob_voxel_map* m, size_t* cols) {
    if (!m || !cols) return fail(OB_INVALID_ARGUMENT, "null pointer");
    *cols = 3 + m->na;
    return OB_OK;
}

ob_status ob_voxel_map_add_points(ob_voxel_map* m, const ob_point_rows* rows, ob_stream* s) {
    if (!m || !rows || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (m->na) return fail(OB_INVALID_ARGUMENT, kDimensionError);
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    Rows r{};
    rs = stage_rows(rows, stg, &r, "stage voxel map rows");
    if (rs != OB_OK || r.cap == 0) return rs;
    return add_batch(m, r, 3, rows->dtype == OB_F64, stg, st);
}

ob_status ob_voxel_map_add_rows(ob_voxel_map* m, const ob_map_rows* rows, ob_stream* s) {
    if (!m || !rows || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (rows->cols != 3 + m->na) return fail(OB_INVALID_ARGUMENT, kDimensionError);
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    Rows r{};
    rs = count_rows(rows->n, rows->n_device, rows->capacity, &r);
    if (rs != OB_OK) return rs;
    if (r.cap && !rows->rows) return fail(OB_INVALID_ARGUMENT, "null rows buffer");
    if (r.cap == 0) return OB_OK;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    r.p = stg.in(rows->rows, r.cap * rows->cols);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage voxel map rows");
    return add_batch(m, r, static_cast<unsigned>(rows->cols), true, stg, st);
}

ob_status ob_voxel_map_remove_far(ob_voxel_map* m, const ob_voxel_map_cull_io* io, ob_stream* s) {
    if (!m || !io || !s || !io->origin) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (io->extracted && !io->n_extracted) return fail(OB_INVALID_ARGUMENT, "extraction needs n_extracted");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    const bool extract = io->n_extracted != nullptr;
    // the kernel writes a device count itself: it is zeroed here only for an empty map or a refused call
    CountedRows res(io->n_extracted, io->extracted ? io->capacity : CountedRows::kCountOnly, stg, st, "voxel map cull");
    const double* org = stg.in(io->origin, 3);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage origin");
    if (!m->slots.cap) return res.zero();
    if (extract) {  // refused before the cull, so a refused call leaves the map as it was
        rs = res.refuse({io->extracted}, kMixedCount);
        if (rs != OB_OK) return rs;
    }
    uint32_t* removed = nullptr;
    if (extract) {
        removed = stg.scratch<uint32_t>(m->slots.cap);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "voxel map cull");
    }
    launch(OB_FAM_VOXEL_MAP, vm_cull_kernel, blocks_for(m->slots.cap), 256, 0, st, table_of(m), counters(m), org,
           m->inv, cull_threshold(m->max_distance, m->inv), removed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "voxel map cull");
    if (!extract) return OB_OK;
    return emit_rows(m, removed, stg, st, io->extracted, io->capacity, res, "voxel map extract");
}

ob_status ob_voxel_map_point_cloud(const ob_voxel_map* m, double* points, size_t capacity, size_t* n_out, ob_stream* s) {
    if (!m || !s || !n_out) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    // as ob_voxel_map_remove_far: a device count is zeroed only for an empty map or a refused call
    CountedRows res(n_out, points ? capacity : CountedRows::kCountOnly, stg, st, "voxel map point cloud");
    if (!m->slots.cap) return res.zero();
    rs = res.refuse({points}, kMixedCount);
    if (rs != OB_OK) return rs;
    return emit_rows(m, nullptr, stg, st, points, capacity, res, "voxel map point cloud");
}

ob_status ob_voxel_map_size(const ob_voxel_map* m, size_t* voxels, size_t* points, ob_stream* s) {
    if (!m || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    unsigned long long c[C_WORDS] = {};
    cudaError_t e = cudaMemcpyAsync(c, counters(m), sizeof(c), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "voxel map size");
    if (c[C_FULL]) return fail(OB_RUNTIME_ERROR, "voxel map table overflow");
    if (voxels) *voxels = static_cast<size_t>(c[C_LIVE]);
    if (points) *points = static_cast<size_t>(c[C_POINTS]);
    return OB_OK;
}

ob_status ob_voxel_map_closest_neighbors(const ob_voxel_map* m, const ob_voxel_query_io* io, ob_stream* s) {
    if (!m || !io || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    Rows r{};
    rs = stage_rows(&io->queries, stg, &r, "stage queries");
    if (rs != OB_OK || r.cap == 0) return rs;
    if (!io->neighbors) return fail(OB_INVALID_ARGUMENT, "null neighbors buffer");
    double* nb = stg.out(io->neighbors, r.cap * (3 + m->na));
    double* d2 = stg.out(io->distances_sq, r.cap);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage neighbors");
    const Table t = table_of(m);
    const bool f64 = io->queries.dtype == OB_F64, attr = m->na != 0;
    auto kern = f64 ? (attr ? vm_closest_kernel<double, true> : vm_closest_kernel<double, false>)
                    : (attr ? vm_closest_kernel<float, true> : vm_closest_kernel<float, false>);
    launch(OB_FAM_VOXEL_MAP, kern, blocks_for(r.cap), 256, 0, st, r, t, m->inv, m->voxel_size, io->max_distance_sq, nb,
           d2);
    stg.check(cudaGetLastError());
    cudaError_t e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "voxel map closest neighbors");
    return OB_OK;
}

ob_status ob_icp_linear_system(const ob_icp_system_io* io, ob_stream* s) {
    if (!io || !s || !io->jtj || !io->jtr) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    Rows r{};
    rs = count_rows(io->n, io->n_device, io->capacity, &r, "too many pairs in one call");
    if (rs != OB_OK) return rs;
    const size_t cap = r.cap;
    if (cap && (!io->source || !io->target)) return fail(OB_INVALID_ARGUMENT, "null pairs buffer");
    const double* src = stg.in(io->source, cap * 3);
    const double* tgt = stg.in(io->target, cap * 3);
    double* jtj = stg.out(io->jtj, 36);
    double* jtr = stg.out(io->jtr, 6);
    // a host count travels by value as the clamp (cap == n), a device count is read by the kernels
    const unsigned long long* n = r.n_dev;
    const unsigned slots = tree_slots(cap);
    double* val = stg.scratch<double>(static_cast<size_t>(slots) * kSys);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage linear system");
    launch(OB_FAM_ICP, icp_leaf_kernel, blocks_for(slots), 256, 0, st, src, tgt, n, cap, io->kernel_scale, nullptr,
           slots, val);
    launch(OB_FAM_ICP, icp_system_kernel, 1, kTreeThreads, 0, st, n, cap, val, jtj, jtr);
    stg.check(cudaGetLastError());
    cudaError_t e = stg.finish();
    if (e != cudaSuccess) return fail_cuda(e, "icp linear system");
    return OB_OK;
}

ob_status ob_icp_align(const ob_voxel_map* m, const ob_icp_io* io, ob_stream* s) {
    if (!m || !io || !s || !io->pose) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    Rows r{};
    rs = stage_rows(&io->source, stg, &r, "stage icp source");
    if (rs != OB_OK) return rs;
    auto* state = stg.scratch<IcpState>(1);
    double* pose = stg.out(io->pose, 16);
    int32_t* iters = stg.out(io->iterations, 1);
    const unsigned cap = std::max(r.cap, 1u);
    const unsigned nb = (cap + kAssocThreads - 1) / kAssocThreads;
    const unsigned slots = tree_slots(cap);
    auto* src = stg.scratch<double>(cap * 3ull);
    auto* tgt = stg.scratch<double>(cap * 3ull);
    auto* ps = stg.scratch<double>(cap * 3ull);
    auto* pt = stg.scratch<double>(cap * 3ull);
    auto* valid = stg.scratch<uint32_t>(cap);
    auto* bc = stg.scratch<uint32_t>(nb);
    auto* val = stg.scratch<double>(static_cast<size_t>(slots) * kSys);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "icp workspace");
    const Table t = table_of(m);
    const double md2 = io->max_distance * io->max_distance;  // square(max_correspondance_distance)
    const double crit_sq = io->convergence_criterion * io->convergence_criterion;
    if (io->source.dtype == OB_F64)
        launch(OB_FAM_ICP, icp_init_kernel<double>, nb, kAssocThreads, 0, st, r, counters(m), src, state);
    else
        launch(OB_FAM_ICP, icp_init_kernel<float>, nb, kAssocThreads, 0, st, r, counters(m), src, state);
    for (int it = 0; it < io->max_num_iterations; ++it) {
        launch(OB_FAM_ICP, icp_assoc_kernel, nb, kAssocThreads, 0, st, r, t, m->inv, m->voxel_size, md2, src, tgt,
               valid, bc, state);
        launch(OB_FAM_ICP, icp_compact_kernel, nb, kAssocThreads, 0, st, r.cap, src, tgt, valid, bc, ps, pt, state);
        launch(OB_FAM_ICP, icp_leaf_kernel, blocks_for(slots), 256, 0, st, ps, pt, &state->n_pairs, cap,
               io->kernel_scale, &state->done, slots, val);
        launch(OB_FAM_ICP, icp_solve_kernel, 1, kTreeThreads, 0, st, val, crit_sq, state);
    }
    launch(OB_FAM_ICP, icp_finish_kernel, 1, 1, 0, st, state, pose, iters);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "icp launch");
    e = stg.finish();  // host pose / iterations: one wait; device ones: nothing waits for the GPU
    if (e != cudaSuccess) return fail_cuda(e, "icp result");
    return OB_OK;
}

}  // extern "C"
