// ob_zone.cu -- zone monitoring (DESIGN f-8): Zone::render of a whole zone set into near/far range images, and
// the per-frame occupancy of EmulatedZoneMon over a device-resident monitor.
//
// Render restates, operation for operation in float with no contraction, Triangle::intersect
// (ouster_core/src/triangle.cpp:19-50), the bounding-sphere test and the multiset of Mesh
// (mesh.cpp:249-294) and the rounding of Zone::render (zone.cpp:102-125).  A multiset reduces to (hits capped
// at 2, min t, max t): its size decides the case and its ends are the result.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "ob_api_common.h"
#include "ob_arith.cuh"

struct ob_zone_monitor {
    int device;
    uint32_t h, w, n_live;
    ob::DeviceBlock near_mm, far_mm;  // uint32 n_live x h x w
    ob::DeviceBlock acc;              // ZoneAcc[OB_ZONE_MAX_LIVE]
    ob::DeviceBlock ctl;              // ZoneCtl[OB_ZONE_MAX_LIVE]
    ob::DeviceBlock states;           // ob_zone_state[OB_ZONE_MAX_LIVE]
};

namespace ob {
namespace {

constexpr int kRenderThreads = 256;
constexpr int kRenderPx = 2;  // pixels per thread
constexpr int kRenderTile = kRenderThreads * kRenderPx;
constexpr float kEps = FLT_EPSILON;  // std::numeric_limits<float>::epsilon()

struct ZoneGpu {
    float cx, cy, cz, radius;  // Mesh::bounding_sphere()
    uint32_t n_tri;
    uint32_t tri_off;  // first triangle in the packed (v0, e1, e2) array
    int32_t body;      // 1: the LUT with sensor_to_body
    int32_t pad;
};

struct V3 {
    float x, y, z;
};
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)}; }
// Eigen's cross: (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)
__device__ __forceinline__ V3 cross3(V3 a, V3 b) {
    return {__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)), __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
            __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
// Eigen's 3-term dot: (x0 y0 + x1 y1) + x2 y2
__device__ __forceinline__ float dot3(V3 a, V3 b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}

// Triangle::intersect with edge1 = v1 - v0 and edge2 = v2 - v0 formed once per zone (the same float
// subtractions the reference repeats per call).  The comparisons are the reference's, unnegated, so a NaN
// passes every rejection and comes out as a NaN t, which `t > 0` never counts.
__device__ __forceinline__ float tri_intersect(V3 o, V3 d, V3 v0, V3 e1, V3 e2) {
    const V3 rc = cross3(d, e2);
    const float det = dot3(e1, rc);
    if (det > -kEps && det < kEps) return -FLT_MAX;
    const float inv = __frcp_rn(det);
    const V3 s = sub3(o, v0);
    const float u = __fmul_rn(inv, dot3(s, rc));
    if ((u < 0.f && fabsf(u) > kEps) || (u > 1.f && fabsf(__fsub_rn(u, 1.f)) > kEps)) return -FLT_MAX;
    const V3 sc = cross3(s, e1);
    const float v = __fmul_rn(inv, dot3(d, sc));
    const float uv = __fadd_rn(u, v);
    if ((v < 0.f && fabsf(v) > kEps) || (uv > 1.f && fabsf(__fsub_rn(uv, 1.f)) > kEps)) return -FLT_MAX;
    return __fmul_rn(inv, dot3(e2, sc));
}

// Mesh::intersects_with_bounding_sphere (mesh.cpp:249-266)
__device__ __forceinline__ bool sphere_hit(const ZoneGpu& z, V3 o, V3 d) {
    const V3 oc = sub3(o, V3{z.cx, z.cy, z.cz});
    const float b = dot3(oc, d);
    const float c = __fsub_rn(dot3(oc, oc), __fmul_rn(z.radius, z.radius));
    if (c > 0.0f && b > 0.0f) return false;
    return __fsub_rn(__fmul_rn(b, b), c) >= 0.0f;
}

// grid (pixel tiles, zones).  A tile whose rays all miss the zone's bounding sphere never stages the mesh.
__global__ void __launch_bounds__(kRenderThreads) zone_render_kernel(
    const ZoneGpu* __restrict__ zones, const float* __restrict__ tris, const double* __restrict__ bdir,
    const double* __restrict__ boff, const double* __restrict__ sdir, const double* __restrict__ soff, uint32_t npx,
    uint32_t* __restrict__ near_mm, uint32_t* __restrict__ far_mm, uint32_t* __restrict__ hits,
    uint32_t* __restrict__ overflow) {
    extern __shared__ float s_tri[];  // n_tri x 9: v0, e1, e2
    const uint32_t zi = blockIdx.y;
    const ZoneGpu z = zones[zi];
    const double* dir = z.body ? bdir : sdir;
    const double* off = z.body ? boff : soff;
    V3 o[kRenderPx], d[kRenderPx];
    bool live[kRenderPx];
    bool any = false;
#pragma unroll
    for (int k = 0; k < kRenderPx; ++k) {
        const uint32_t p = blockIdx.x * kRenderTile + k * kRenderThreads + threadIdx.x;
        live[k] = false;
        if (p < npx) {
            // beam.offset = offset.cast<float>(); beam.direction = direction.cast<float>() * 1000.0f
            o[k] = {__double2float_rn(off[3 * p]), __double2float_rn(off[3 * p + 1]), __double2float_rn(off[3 * p + 2])};
            d[k] = {__fmul_rn(__double2float_rn(dir[3 * p]), 1000.0f), __fmul_rn(__double2float_rn(dir[3 * p + 1]), 1000.0f),
                    __fmul_rn(__double2float_rn(dir[3 * p + 2]), 1000.0f)};
            live[k] = sphere_hit(z, o[k], d[k]);
            any = any || live[k];
        }
    }
    uint32_t n_hit[kRenderPx] = {};
    float t_min[kRenderPx], t_max[kRenderPx];
#pragma unroll
    for (int k = 0; k < kRenderPx; ++k) t_min[k] = INFINITY, t_max[k] = 0.0f;
    if (__syncthreads_or(any)) {
        const float* src = tris + size_t(z.tri_off) * 9;
        for (uint32_t i = threadIdx.x; i < z.n_tri * 9; i += kRenderThreads) s_tri[i] = src[i];
        __syncthreads();
        for (uint32_t t = 0; t < z.n_tri; ++t) {
            const float* q = s_tri + 9 * t;
            const V3 v0{q[0], q[1], q[2]}, e1{q[3], q[4], q[5]}, e2{q[6], q[7], q[8]};
#pragma unroll
            for (int k = 0; k < kRenderPx; ++k) {
                if (!live[k]) continue;
                const float dist = tri_intersect(o[k], d[k], v0, e1, e2);
                if (dist > 0) {
                    n_hit[k] = min(n_hit[k] + 1u, 2u);
                    t_min[k] = fminf(t_min[k], dist);
                    t_max[k] = fmaxf(t_max[k], dist);
                }
            }
        }
    }
    uint32_t px_hits = 0;
#pragma unroll
    for (int k = 0; k < kRenderPx; ++k) {
        const uint32_t p = blockIdx.x * kRenderTile + k * kRenderThreads + threadIdx.x;
        if (p >= npx) continue;
        // closest_and_farthest_intersections: >= 2 hits (min, max), 1 hit (0, t), none (0, 0)
        float nf = 0.f, ff = 0.f;
        if (live[k] && n_hit[k] >= 1) {
            ++px_hits;
            ff = t_max[k];
            nf = n_hit[k] >= 2 ? t_min[k] : 0.f;
        }
        const double nm = round(__dmul_rn(double(nf), 1000.0));
        const double fm = round(__dmul_rn(double(ff), 1000.0));
        const bool ovf = nm > 4294967295.0 || fm > 4294967295.0;
        if (ovf) atomicOr(overflow + zi, 1u);
        near_mm[size_t(zi) * npx + p] = ovf ? 0u : uint32_t(nm);
        far_mm[size_t(zi) * npx + p] = ovf ? 0u : uint32_t(fm);
    }
    const uint32_t warp_hits = __reduce_add_sync(0xffffffffu, px_hits);
    if ((threadIdx.x & 31) == 0 && warp_hits) atomicAdd(hits + zi, warp_hits);
}

// ---- occupancy ----
constexpr int kOccThreads = 256;
constexpr int kOccPx = 4;
constexpr int kOccTile = kOccThreads * kOccPx;

struct ZoneAcc {
    uint32_t count, occlusion, invalid, min_r, max_r, pad;
    unsigned long long sum;
};
struct ZoneCtl {
    uint32_t id, mode, point_count, frame_count, triggers, alerts, max_count, pad;
    unsigned long long range_sum;  // exact sum of the last update's triggering ranges
};

__global__ void zone_acc_reset_kernel(ZoneAcc* acc) {
    if (threadIdx.x < OB_ZONE_MAX_LIVE) acc[threadIdx.x] = ZoneAcc{0, 0, 0, 0xffffffffu, 0, 0, 0};
}

// max_count = #(near < far) per zone, once per monitor
__global__ void zone_max_count_kernel(const uint32_t* __restrict__ near_mm, const uint32_t* __restrict__ far_mm,
                                      uint32_t npx, ZoneCtl* ctl) {
    const uint32_t z = blockIdx.y;
    uint32_t c = 0;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < npx; p += gridDim.x * blockDim.x)
        c += near_mm[size_t(z) * npx + p] < far_mm[size_t(z) * npx + p];
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&ctl[z].max_count, c);
}

// _calc_counts (zone_common.py:47-78): integer counts and atomics, so the result does not depend on scheduling
__global__ void __launch_bounds__(kOccThreads) zone_occupancy_kernel(
    const uint32_t* __restrict__ range, const uint32_t* __restrict__ near_mm, const uint32_t* __restrict__ far_mm,
    uint32_t n_live, uint32_t npx, ZoneAcc* __restrict__ acc, uint32_t* __restrict__ bitmask) {
    __shared__ ZoneAcc s_acc[OB_ZONE_MAX_LIVE];
    if (threadIdx.x < OB_ZONE_MAX_LIVE) s_acc[threadIdx.x] = ZoneAcc{0, 0, 0, 0xffffffffu, 0, 0, 0};
    __syncthreads();
    uint32_t r[kOccPx], bits[kOccPx];
#pragma unroll
    for (int k = 0; k < kOccPx; ++k) {
        const uint32_t p = blockIdx.x * kOccTile + k * kOccThreads + threadIdx.x;
        r[k] = p < npx ? range[p] : 0u;
        bits[k] = 0;
    }
    for (uint32_t z = 0; z < n_live; ++z) {
        uint32_t cnt = 0, occ = 0, inv = 0, mn = 0xffffffffu, mx = 0;
        unsigned long long sum = 0;
#pragma unroll
        for (int k = 0; k < kOccPx; ++k) {
            const uint32_t p = blockIdx.x * kOccTile + k * kOccThreads + threadIdx.x;
            if (p >= npx) continue;
            const uint32_t nr = near_mm[size_t(z) * npx + p], fr = far_mm[size_t(z) * npx + p];
            const bool trig = r[k] > 0 && nr <= r[k] && r[k] <= fr;
            occ += r[k] > 0 && r[k] <= nr;
            inv += r[k] == 0 && nr > 0;
            if (trig) {
                bits[k] |= 1u << z;
                ++cnt;
                sum += r[k];
                mn = min(mn, r[k]);
                mx = max(mx, r[k]);
            }
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        occ = __reduce_add_sync(0xffffffffu, occ);
        inv = __reduce_add_sync(0xffffffffu, inv);
        mn = __reduce_min_sync(0xffffffffu, mn);
        mx = __reduce_max_sync(0xffffffffu, mx);
        sum = warp_sum_u64(sum);
        if ((threadIdx.x & 31) == 0) {
            if (cnt) {
                atomicAdd(&s_acc[z].count, cnt);
                atomicAdd(&s_acc[z].sum, sum);
                atomicMin(&s_acc[z].min_r, mn);
                atomicMax(&s_acc[z].max_r, mx);
            }
            if (occ) atomicAdd(&s_acc[z].occlusion, occ);
            if (inv) atomicAdd(&s_acc[z].invalid, inv);
        }
    }
    __syncthreads();
    if (threadIdx.x < n_live) {
        const ZoneAcc a = s_acc[threadIdx.x];
        ZoneAcc* g = acc + threadIdx.x;
        if (a.count) {
            atomicAdd(&g->count, a.count);
            atomicAdd(&g->sum, a.sum);
            atomicMin(&g->min_r, a.min_r);
            atomicMax(&g->max_r, a.max_r);
        }
        if (a.occlusion) atomicAdd(&g->occlusion, a.occlusion);
        if (a.invalid) atomicAdd(&g->invalid, a.invalid);
    }
    if (bitmask) {
#pragma unroll
        for (int k = 0; k < kOccPx; ++k) {
            const uint32_t p = blockIdx.x * kOccTile + k * kOccThreads + threadIdx.x;
            if (p < npx && bits[k]) bitmask[p] |= bits[k];
        }
    }
}

// calc_triggers' state machine (zone_common.py:86-105) and get_packet (:114-136); leaves the accumulators reset
// for the next update
__global__ void zone_tail_kernel(ZoneAcc* acc, ZoneCtl* ctl, uint32_t n_live, ob_zone_state* states) {
    if (threadIdx.x != 0) return;
    for (uint32_t i = 0; i < OB_ZONE_MAX_LIVE; ++i) {
        ob_zone_state st{};
        if (i < n_live) {
            const ZoneAcc a = acc[i];
            ZoneCtl c = ctl[i];
            const bool trig = (a.count >= c.point_count && c.mode == OB_ZONE_MODE_OCCUPANCY) ||
                              (a.count < c.point_count && c.mode == OB_ZONE_MODE_VACANCY);
            c.triggers = trig ? c.triggers + 1 : 0;
            c.alerts = c.triggers >= c.frame_count ? c.alerts + 1 : 0;
            c.range_sum = a.sum;
            ctl[i] = c;
            st.live = 1;
            st.id = uint8_t(c.id);
            st.trigger_type = uint8_t(c.mode);
            st.trigger_status = c.alerts > 0;
            st.triggered_frames = c.alerts;
            st.count = a.count;
            st.occlusion_count = a.occlusion;
            st.invalid_count = a.invalid;
            st.max_count = c.max_count;
            if (a.count) {
                st.min_range = a.min_r;
                st.max_range = a.max_r;
                // numpy's float64 mean of uint32 (exact below 2^53), truncated into the uint32 record
                st.mean_range = uint32_t(__ddiv_rn(double(a.sum), double(a.count)));
            }
            acc[i] = ZoneAcc{0, 0, 0, 0xffffffffu, 0, 0, 0};
        } else {
            st.id = 255;
        }
        states[i] = st;
    }
}

// Mesh's bounding sphere in the reference's float order (mesh.cpp:41-60): sequential centroid sum over
// v0, v1, v2 of each triangle divided by float(3n); running std::max({|v0-c|^2, |v1-c|^2, |v2-c|^2, r2}).
void bounding_sphere(const float* t, uint32_t n, float c[3], float* radius) {
    volatile float acc[3] = {0.f, 0.f, 0.f};  // volatile: keep the sequential float order
    for (uint32_t i = 0; i < n; ++i)
        for (int v = 0; v < 3; ++v)
            for (int k = 0; k < 3; ++k) acc[k] = acc[k] + t[9 * i + 3 * v + k];
    const float denom = float(size_t(3) * n);
    for (int k = 0; k < 3; ++k) c[k] = acc[k] / denom;
    auto sq = [&](const float* p) {
        volatile float dx = p[0] - c[0], dy = p[1] - c[1], dz = p[2] - c[2];
        volatile float xx = dx * dx, yy = dy * dy, zz = dz * dz;
        volatile float s = xx + yy;
        return float(s + zz);
    };
    float r2 = 0.f;
    for (uint32_t i = 0; i < n; ++i) {
        const float a = sq(t + 9 * i), b = sq(t + 9 * i + 3), cc = sq(t + 9 * i + 6);
        float m = a;  // std::max(initializer_list): the first of the largest, by operator<
        if (m < b) m = b;
        if (m < cc) m = cc;
        if (m < r2) m = r2;
        r2 = m;
    }
    *radius = std::sqrt(r2);
}

ob_status check_zone(const ob_zone_desc& z, bool have_body) {
    // Zone::check_invariants (zone.cpp:18-46), then the early returns of Zone::render (:64-85)
    if (z.point_count == 0) return fail(OB_INVALID_ARGUMENT, "Zone: point_count must be in [1, 262143]");
    if (z.frame_count == 0) return fail(OB_INVALID_ARGUMENT, "Zone: frame_count must be in [1, 65535]");
    if (z.mode != OB_ZONE_MODE_OCCUPANCY && z.mode != OB_ZONE_MODE_VACANCY)
        return fail(OB_INVALID_ARGUMENT, "Zone: mode must be OCCUPANCY or VACANCY");
    if (z.coordinate_frame != OB_ZONE_FRAME_BODY && z.coordinate_frame != OB_ZONE_FRAME_SENSOR)
        return fail(OB_INVALID_ARGUMENT, "Zone: STL coordinate frame must be BODY or SENSOR");
    if (z.n_triangles == 0) return fail(OB_INVALID_ARGUMENT, "Zone: Error rendering zone, STL has no triangles.");
    if (z.n_triangles > OB_ZONE_MAX_TRIANGLES)
        return fail(OB_INVALID_ARGUMENT, "Zone: Error rendering zone, STL has too many triangles.");
    if (!z.triangles) return fail(OB_INVALID_ARGUMENT, "null triangles buffer");
    if (z.coordinate_frame == OB_ZONE_FRAME_BODY && !have_body)
        return fail(OB_INVALID_ARGUMENT,
                    "Zone: Error rendering zone, sensor_to_body_transform not set for BODY coordinate frame.");
    return OB_OK;
}

// the 72 KB dynamic shared-memory opt-in is a per-device attribute: set it once on each device that renders
cudaError_t render_smem_opt_in(int device) {
    static std::mutex mx;
    static bool done[64] = {};
    std::lock_guard<std::mutex> lock(mx);
    if (device >= 0 && device < 64 && done[device]) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(zone_render_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         OB_ZONE_MAX_TRIANGLES * 9 * int(sizeof(float)));
    if (e == cudaSuccess && device >= 0 && device < 64) done[device] = true;
    return e;
}

}  // namespace
}  // namespace ob

using namespace ob;

extern "C" {

ob_status ob_zone_render(const ob_zone_render_io* io, ob_stream* s) {
    if (!io || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (io->n_zones && !io->zones) return fail(OB_INVALID_ARGUMENT, "null zones");
    const bool have_body = io->body_direction && io->body_offset;
    for (uint32_t i = 0; i < io->n_zones; ++i) {
        ob_status rs = check_zone(io->zones[i], have_body);
        if (rs != OB_OK) return rs;
    }
    const size_t npx = size_t(io->n_rows) * io->n_cols;
    if (io->n_zones == 0 || npx == 0) return OB_OK;
    if (!io->sensor_direction || !io->sensor_offset) return fail(OB_INVALID_ARGUMENT, "null sensor LUT");
    if (!io->near_mm || !io->far_mm || !io->pixels_with_intersections)
        return fail(OB_INVALID_ARGUMENT, "null output buffer");
    if (npx > 0xffffffffull / 2) return fail(OB_INVALID_ARGUMENT, "zone image too large");
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    // pack (v0, e1 = v1 - v0, e2 = v2 - v0) per triangle and the bounding sphere of each zone, on the host
    std::vector<ZoneGpu> zg(io->n_zones);
    size_t n_tri_all = 0;
    uint32_t max_tri = 0;
    for (uint32_t i = 0; i < io->n_zones; ++i) n_tri_all += io->zones[i].n_triangles;
    std::vector<float> packed(n_tri_all * 9);
    size_t at = 0;
    for (uint32_t i = 0; i < io->n_zones; ++i) {
        const ob_zone_desc& z = io->zones[i];
        float c[3], r;
        bounding_sphere(z.triangles, z.n_triangles, c, &r);
        zg[i] = ZoneGpu{c[0], c[1], c[2], r, z.n_triangles, uint32_t(at), z.coordinate_frame == OB_ZONE_FRAME_BODY, 0};
        for (uint32_t t = 0; t < z.n_triangles; ++t, ++at) {
            const float* v = z.triangles + 9 * size_t(t);
            float* q = packed.data() + 9 * at;
            for (int k = 0; k < 3; ++k) {
                q[k] = v[k];
                q[3 + k] = v[3 + k] - v[k];
                q[6 + k] = v[6 + k] - v[k];
            }
        }
        max_tri = std::max(max_tri, z.n_triangles);
    }
    Staging stg(st);
    stg.check(render_smem_opt_in(device));
    const double* sd = stg.in(io->sensor_direction, npx * 3);
    const double* so = stg.in(io->sensor_offset, npx * 3);
    const double* bd = have_body ? stg.in(io->body_direction, npx * 3) : nullptr;
    const double* bo = have_body ? stg.in(io->body_offset, npx * 3) : nullptr;
    const float* tris = stg.in(packed.data(), packed.size());
    const ZoneGpu* zdev = stg.in(zg.data(), zg.size());
    uint32_t* near = stg.out(io->near_mm, npx * io->n_zones);
    uint32_t* far = stg.out(io->far_mm, npx * io->n_zones);
    uint32_t* hits = stg.scratch<uint32_t>(size_t(io->n_zones) * 2);  // hits, then overflow flags
    cudaError_t e = stg.error();
    if (e == cudaSuccess) e = cudaMemsetAsync(hits, 0, size_t(io->n_zones) * 8, st);
    if (e != cudaSuccess) return fail_cuda(e, "stage zone render");
    uint32_t* ovf = hits + io->n_zones;
    const dim3 grid(unsigned((npx + kRenderTile - 1) / kRenderTile), io->n_zones);
    launch(OB_FAM_ZONE, zone_render_kernel, grid, kRenderThreads, size_t(max_tri) * 9 * sizeof(float), st, zdev, tris,
           bd, bo, sd, so, uint32_t(npx), near, far, hits, ovf);
    std::vector<uint32_t> hf(size_t(io->n_zones) * 2);
    stg.check(cudaGetLastError());
    if (!stg.error()) stg.check(cudaMemcpyAsync(hf.data(), hits, hf.size() * 4, cudaMemcpyDeviceToHost, st));
    e = stg.flush();
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "zone render");
    for (uint32_t i = 0; i < io->n_zones; ++i) {
        io->pixels_with_intersections[i] = hf[i];
        if (hf[io->n_zones + i]) return fail(OB_RUNTIME_ERROR, "Zone::render: range overflow");
        if (hf[i] > 0 && hf[i] < io->zones[i].point_count)
            return fail(OB_RUNTIME_ERROR, "Zone: area of rendered zone (" + std::to_string(hf[i]) +
                                              ") is smaller than point_count (" +
                                              std::to_string(io->zones[i].point_count) + ") specified in zone.");
    }
    return OB_OK;
}

ob_status ob_zone_monitor_create(int device, uint32_t n_rows, uint32_t n_cols, const ob_zone_live* live,
                                 uint32_t n_live, ob_zone_monitor** out) {
    if (!out || (n_live && !live)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    *out = nullptr;
    if (n_live > OB_ZONE_MAX_LIVE) return fail(OB_INVALID_ARGUMENT, "at most 16 live zones");
    const size_t npx = size_t(n_rows) * n_cols;
    if (npx > 0xffffffffull / 2) return fail(OB_INVALID_ARGUMENT, "zone image too large");
    for (uint32_t i = 0; i < n_live; ++i)
        if (npx && (!live[i].near_mm || !live[i].far_mm)) return fail(OB_INVALID_ARGUMENT, "null zone image");
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    std::unique_ptr<ob_zone_monitor> m(new ob_zone_monitor{device, n_rows, n_cols, n_live});
    const size_t img = npx * 4;
    cudaError_t e = m->near_mm.alloc(std::max<size_t>(img * n_live, 4));
    if (e == cudaSuccess) e = m->far_mm.alloc(std::max<size_t>(img * n_live, 4));
    if (e == cudaSuccess) e = m->acc.alloc(sizeof(ZoneAcc) * OB_ZONE_MAX_LIVE);
    if (e == cudaSuccess) e = m->ctl.alloc(sizeof(ZoneCtl) * OB_ZONE_MAX_LIVE);
    if (e == cudaSuccess) e = m->states.alloc(sizeof(ob_zone_state) * OB_ZONE_MAX_LIVE);
    uint32_t* near_mm = m->near_mm.get<uint32_t>();
    uint32_t* far_mm = m->far_mm.get<uint32_t>();
    ZoneCtl ctl[OB_ZONE_MAX_LIVE] = {};
    for (uint32_t i = 0; i < n_live; ++i) {
        ctl[i] = ZoneCtl{live[i].id, uint32_t(live[i].mode), live[i].point_count, live[i].frame_count,
                         live[i].triggers, live[i].alerts, 0, 0, 0};
        if (e == cudaSuccess && img) e = cudaMemcpy(near_mm + i * npx, live[i].near_mm, img, cudaMemcpyDefault);
        if (e == cudaSuccess && img) e = cudaMemcpy(far_mm + i * npx, live[i].far_mm, img, cudaMemcpyDefault);
    }
    if (e == cudaSuccess) e = cudaMemcpy(m->ctl.get(), ctl, sizeof(ctl), cudaMemcpyHostToDevice);
    // states before the first update: what get_packet() gives for slots that have not been computed
    ob_zone_state st0[OB_ZONE_MAX_LIVE] = {};
    for (uint32_t i = n_live; i < OB_ZONE_MAX_LIVE; ++i) st0[i].id = 255;
    if (e == cudaSuccess) e = cudaMemcpy(m->states.get(), st0, sizeof(st0), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        launch(OB_FAM_ZONE, zone_acc_reset_kernel, 1, 32, 0, 0, m->acc.get<ZoneAcc>());
        if (n_live && npx) {
            const dim3 grid(unsigned(std::min<size_t>((npx + 255) / 256, 1024)), n_live);
            launch(OB_FAM_ZONE, zone_max_count_kernel, grid, 256, 0, 0, near_mm, far_mm, uint32_t(npx),
                   m->ctl.get<ZoneCtl>());
        }
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return fail_cuda(e, "ob_zone_monitor_create");
    *out = m.release();
    return OB_OK;
}

ob_status ob_zone_monitor_update(ob_zone_monitor* m, const uint32_t* range, uint32_t* bitmask, ob_stream* s) {
    if (!m || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const size_t npx = size_t(m->h) * m->w;
    if (npx && !range) return fail(OB_INVALID_ARGUMENT, "null range");
    if (stream_device(s) != m->device) return fail(OB_INVALID_ARGUMENT, "stream and monitor are on different devices");
    ob_status rs = require_device(m->device);  // the launches below go to the current device
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    const uint32_t* r = stg.in(range, npx);
    const bool host_bm = bitmask && !is_device_ptr(bitmask);
    // a host bitmask is read, OR-ed on the device and copied back
    uint32_t* bm = npx ? stg.inout(bitmask, npx) : nullptr;
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage zone update");
    if (npx)
        launch(OB_FAM_ZONE, zone_occupancy_kernel, unsigned((npx + kOccTile - 1) / kOccTile), kOccThreads, 0, st, r,
               m->near_mm.get<uint32_t>(), m->far_mm.get<uint32_t>(), m->n_live, uint32_t(npx), m->acc.get<ZoneAcc>(),
               bm);
    launch(OB_FAM_ZONE, zone_tail_kernel, 1, 32, 0, st, m->acc.get<ZoneAcc>(), m->ctl.get<ZoneCtl>(), m->n_live,
           m->states.get<ob_zone_state>());
    stg.check(cudaGetLastError());
    cudaError_t e = stg.flush();
    if (e == cudaSuccess && (host_bm || (npx && !is_device_ptr(range)))) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "zone update");
    return OB_OK;
}

ob_status ob_zone_monitor_states(const ob_zone_monitor* m, void* out, ob_stream* s) {
    if (!m || !out || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    const bool dev = is_device_ptr(out);
    cudaError_t e = cudaMemcpyAsync(out, m->states.get(), sizeof(ob_zone_state) * OB_ZONE_MAX_LIVE,
                                    dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && !dev) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "zone states");
    return OB_OK;
}

ob_status ob_zone_monitor_counters(const ob_zone_monitor* m, uint32_t* triggers, uint32_t* alerts,
                                   uint64_t* range_sums, ob_stream* s) {
    if (!m || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(m->device);
    if (rs != OB_OK) return rs;
    ZoneCtl ctl[OB_ZONE_MAX_LIVE];
    cudaStream_t st = stream_handle(s);
    cudaError_t e = cudaMemcpyAsync(ctl, m->ctl.get(), sizeof(ctl), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail_cuda(e, "zone counters");
    for (uint32_t i = 0; i < m->n_live; ++i) {
        if (triggers) triggers[i] = ctl[i].triggers;
        if (alerts) alerts[i] = ctl[i].alerts;
        if (range_sums) range_sums[i] = ctl[i].range_sum;
    }
    return OB_OK;
}

ob_status ob_zone_monitor_destroy(ob_zone_monitor* m) {
    if (!m) return OB_OK;
    DeviceScope on(m->device);
    delete m;
    return OB_OK;
}

}  // extern "C"
