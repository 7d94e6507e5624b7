// ob_normals.cu -- surface normals on destaggered XYZ (SURVEY 8f-2), one thread per pixel.
//
// What it replaces (reference paths relative to /root/reference):
//   compute_vertical_subtent   ouster_algorithm/src/normals.cpp:32-76
//   compute_unit_normals       ouster_algorithm/src/normals.cpp:78-407
//   normals(...) x2            ouster_algorithm/src/normals.cpp:411-483, include/ouster/algorithm/normals.h:58-108
//
// The reference precomputes a normalised beam per pixel and then walks 32x32 tiles on one core; every
// pixel's result depends only on its own beam and on the XYZ/range of the <= 2*search neighbours on
// each axis (both returns), so the whole thing is a stencil: one pass, each pixel read ~5 times from
// L1/L2, written once.  It consumes K1's `xyz_destaggered` / `range_destaggered` outputs in place, so
// range -> destagger -> XYZ -> normals never leaves HBM.
//
// Arithmetic: double, one rounding per operation (explicit __dmul_rn/__dadd_rn: no FMA contraction),
// 3-term reductions as (x0 + x1) + x2 -- the same choices as oracle/orc_normals.c, so results are
// bit-identical to the oracle for double inputs.  Float inputs are widened, results rounded once.
// The vertical pixel subtent needs one acos(); the device's differs from glibc's by at most an ulp
// or two, so it is returned to the caller (tests feed it back to the oracle).
#include <math_constants.h>

#include <algorithm>
#include <cmath>

#include "ob_api_common.h"
#include "ob_arith.cuh"

namespace ob {

namespace {

constexpr double kEps = 2.220446049250313e-16;  // std::numeric_limits<double>::epsilon()
constexpr long long kForegroundSalienceMm = 500;  // normals.cpp:24

struct NormalsParams {
    const void* xyz[2];        // per return: n_frames x (H*W) x 3 of T, destaggered
    const uint32_t* range[2];  // per return: n_frames x H x W
    void* out[2];              // per return: normals, same layout as xyz
    const double* origins;     // W x 3 per frame (stride origins_fs) or null = zeros
    double* subtent[2];        // per return: n_frames doubles (device), the vertical pixel subtent derived from it
    unsigned long long xyz_fs, range_fs, out_fs, origins_fs;  // frame strides in elements
    unsigned H, W, n_frames, search;
    double desired_sq, tan_safe, h_subtent, subtent_override;
    int dual;
};

template <typename T>
__device__ __forceinline__ void load3(const T* base, size_t idx, double (&v)[3]) {
    const T* p = base + idx * 3;
    v[0] = static_cast<double>(p[0]);
    v[1] = static_cast<double>(p[1]);
    v[2] = static_cast<double>(p[2]);
}

// normalised beam of a pixel (normals.cpp:111-129)
template <typename T>
__device__ __forceinline__ void beam_of(const T* xyz, const double* origins, unsigned W, unsigned row, unsigned col,
                                        double (&out)[3]) {
    double d[3];
    load3(xyz, static_cast<size_t>(row) * W + col, d);
    if (origins != nullptr) {
        d[0] = sub(d[0], origins[col * 3 + 0]);
        d[1] = sub(d[1], origins[col * 3 + 1]);
        d[2] = sub(d[2], origins[col * 3 + 2]);
    }
    const double mag = sqrt(dot3(d, d));
    if (mag > 0.0) {
        out[0] = d[0] / mag;
        out[1] = d[1] / mag;
        out[2] = d[2] / mag;
    } else {
        out[0] = out[1] = out[2] = 0.0;
    }
}

// compute_vertical_subtent (normals.cpp:32-76): candidates are visited in the reference's order
// (mid, mid, mid-1, mid+1, ...); a warp examines 32 of them at a time, the first hit in that order wins.
// Warp r of block f derives the subtent of return r of frame f (warp 1 only runs for dual returns).
template <typename T>
__global__ void normals_subtent_kernel(const __grid_constant__ NormalsParams p) {
    const unsigned f = blockIdx.x;
    const unsigned lane = threadIdx.x & 31;
    const unsigned ret = threadIdx.x >> 5;
    const T* xyz = static_cast<const T*>(p.xyz[ret]) + f * p.xyz_fs;
    const uint32_t* range = p.range[ret] + f * p.range_fs;
    const double* origins = p.origins ? p.origins + f * p.origins_fs : nullptr;
    double* subtent = p.subtent[ret];
    const unsigned W = p.W, H = p.H;
    if (p.subtent_override > 0.0) {
        if (lane == 0) subtent[f] = p.subtent_override;
        return;
    }
    const unsigned mid = W / 2;
    const unsigned n_cand = 2 * (mid + 1);
    for (unsigned base = 0; base < n_cand; base += 32) {
        const unsigned i = base + lane;
        bool found = false;
        double value = 0.0;
        if (i < n_cand) {
            const int off = static_cast<int>(i / 2);
            const int col_i = static_cast<int>(mid) + ((i & 1u) ? off : -off);
            if (col_i >= 0 && col_i < static_cast<int>(W)) {
                const unsigned col = static_cast<unsigned>(col_i);
                unsigned top = H > 0 ? H - 1 : 0, bottom = 0;
                while (top > bottom) {
                    const bool ht = range[static_cast<size_t>(top) * W + col] != 0;
                    const bool hb = range[static_cast<size_t>(bottom) * W + col] != 0;
                    if (ht && hb) {
                        double vt[3], vb[3];
                        beam_of(xyz, origins, W, top, col, vt);
                        beam_of(xyz, origins, W, bottom, col, vb);
                        double dp = dot3(vt, vb);
                        dp = fmax(-1.0, fmin(1.0, dp));
                        value = acos(dp) / static_cast<double>(top - bottom);
                        found = true;
                        break;
                    }
                    top -= ht ? 0u : 1u;
                    bottom += hb ? 0u : 1u;
                }
            }
        }
        const unsigned mask = __ballot_sync(0xffffffffu, found);
        if (mask != 0) {
            const int src = __ffs(mask) - 1;
            const double v = __shfl_sync(0xffffffffu, value, src);
            if (lane == 0) subtent[f] = v;
            return;
        }
    }
    if (lane == 0) {  // no valid pair: 90 degrees of vertical field of view over the image height
        const unsigned long long hm1 = static_cast<unsigned long long>(H) - 1ull;  // size_t arithmetic of the reference
        const unsigned long long intervals = hm1 > 1ull ? hm1 : 1ull;
        subtent[f] = (0.5 * 3.14159265358979323846) / static_cast<double>(intervals);
    }
}

struct Best {
    double diff[3];
    double min_sq;
    unsigned radius;
    bool flip, thin;
};

// consider_neighbor (normals.cpp:177-205)
template <typename T>
__device__ __forceinline__ void consider(const T* xyz_base, const uint32_t* rng_base, size_t idx, bool flip,
                                         unsigned radius, const double (&center)[3], uint32_t center_range,
                                         double desired_sq, Best& s) {
    const uint32_t nr = rng_base[idx];
    if (nr == 0) return;
    double nv[3];
    load3(xyz_base, idx, nv);
    const double diff[3] = {sub(nv[0], center[0]), sub(nv[1], center[1]), sub(nv[2], center[2])};
    const double dsq = dot3(diff, diff);
    if (static_cast<long long>(nr) - static_cast<long long>(center_range) < kForegroundSalienceMm) s.thin = false;
    if (fabs(sub(dsq, desired_sq)) < fabs(sub(s.min_sq, desired_sq))) {
        s.diff[0] = diff[0];
        s.diff[1] = diff[1];
        s.diff[2] = diff[2];
        s.min_sq = dsq;
        s.flip = flip;
        s.radius = radius;
    }
}

// find_best_neighbor (normals.cpp:157-268)
template <typename T, bool VERTICAL>
__device__ __forceinline__ bool find_best(const NormalsParams& p, const T* xyz, const uint32_t* range, const T* xyz2,
                                          const uint32_t* range2, unsigned row, unsigned col, double neighbor_sq,
                                          const double (&center)[3], uint32_t center_range, double (&diff)[3],
                                          bool& flip, bool& thin, unsigned max_up, unsigned max_down) {
    Best s;
    s.diff[0] = s.diff[1] = s.diff[2] = 0.0;
    s.min_sq = CUDART_INF;
    s.radius = 1;
    s.flip = false;
    s.thin = thin;
    bool good = false;
    const unsigned W = p.W;
    for (unsigned radius = 1; radius <= p.search; ++radius) {
        if (VERTICAL && radius > max_up && radius > max_down) break;
        if (good && !s.thin) break;
        if (VERTICAL) {
            const size_t up = static_cast<size_t>(row - radius) * W + col, down = static_cast<size_t>(row + radius) * W + col;
            if (radius <= max_up) consider(xyz, range, up, true, radius, center, center_range, p.desired_sq, s);
            if (radius <= max_down) consider(xyz, range, down, false, radius, center, center_range, p.desired_sq, s);
            if (p.dual) {
                if (radius <= max_up) consider(xyz2, range2, up, true, radius, center, center_range, p.desired_sq, s);
                if (radius <= max_down) consider(xyz2, range2, down, false, radius, center, center_range, p.desired_sq, s);
            }
        } else {
            const int wi = static_cast<int>(W);
            const int lu = static_cast<int>(col) - static_cast<int>(radius);
            const size_t left = static_cast<size_t>(row) * W + static_cast<unsigned>(((lu % wi) + wi) % wi);
            const size_t right = static_cast<size_t>(row) * W +
                                 static_cast<unsigned>((static_cast<int>(col) + static_cast<int>(radius)) % wi);
            consider(xyz, range, left, true, radius, center, center_range, p.desired_sq, s);
            if (p.dual) consider(xyz2, range2, left, true, radius, center, center_range, p.desired_sq, s);
            consider(xyz, range, right, false, radius, center, center_range, p.desired_sq, s);
            if (p.dual) consider(xyz2, range2, right, false, radius, center, center_range, p.desired_sq, s);
        }
        const double lim = mul(mul(static_cast<double>(s.radius), static_cast<double>(s.radius)), neighbor_sq);
        if (p.desired_sq <= s.min_sq && s.min_sq < lim) {
            good = true;
        } else if (radius == p.search) {
            if (s.min_sq > 0 && s.min_sq < lim) good = true;
        }
    }
    thin = s.thin;
    if (good && s.min_sq < CUDART_INF) {
        diff[0] = s.diff[0];
        diff[1] = s.diff[1];
        diff[2] = s.diff[2];
        flip = s.flip;
        return true;
    }
    return false;
}

// compute_unit_normals (normals.cpp:270-406) for return `ret` (the other return supplies extra neighbours)
template <typename T>
__global__ void __launch_bounds__(256) normals_kernel(const __grid_constant__ NormalsParams p, int ret) {
    const unsigned v = blockIdx.x * 32 + (threadIdx.x & 31);
    const unsigned u = blockIdx.y * 8 + (threadIdx.x >> 5);
    const unsigned f = blockIdx.z;
    if (u >= p.H || v >= p.W) return;
    const int other = ret ^ 1;
    const T* xyz = static_cast<const T*>(p.xyz[ret]) + f * p.xyz_fs;
    const uint32_t* range = p.range[ret] + f * p.range_fs;
    const T* xyz2 = p.dual ? static_cast<const T*>(p.xyz[other]) + f * p.xyz_fs : nullptr;
    const uint32_t* range2 = p.dual ? p.range[other] + f * p.range_fs : nullptr;
    const double* origins = p.origins ? p.origins + f * p.origins_fs : nullptr;
    T* out = static_cast<T*>(p.out[ret]) + f * p.out_fs;
    const size_t idx = static_cast<size_t>(u) * p.W + v;
    double n[3] = {0.0, 0.0, 0.0};
    const uint32_t cr = range[idx];
    do {
        if (cr == 0) break;
        double center[3], beam[3];
        load3(xyz, idx, center);
        beam_of(xyz, origins, p.W, u, v, beam);
        if (dot3(beam, beam) <= kEps) break;
        // The dual-return overload passes the first return's subtent to both passes, but
        // compute_unit_normals only honours an override > 0 (normals.cpp:134-140, 447-479): when the
        // first return's subtent is 0, the second return's pass derives its own from (xyz2, range2).
        double v_subtent = p.subtent[0][f];
        if (ret == 1 && !(v_subtent > 0.0)) v_subtent = p.subtent[1][f];
        // calc_max_distance_threshold (normals.cpp:143-151)
        const double two_pi = 2.0 * 3.14159265358979323846;
        const double perimeter = mul(two_pi, mul(static_cast<double>(cr), 0.001));
        const double nh = (perimeter / (two_pi / p.h_subtent)) / p.tan_safe;
        const double nv = (perimeter / (two_pi / v_subtent)) / p.tan_safe;
        const unsigned max_up = min(p.search, u), max_down = min(p.search, p.H - 1 - u);
        double vd[3] = {0, 0, 0}, hd[3] = {0, 0, 0};
        bool vflip = false, hflip = false, vthin = true, hthin = true;
        const bool vfound = find_best<T, true>(p, xyz, range, xyz2, range2, u, v, mul(nv, nv), center, cr, vd, vflip,
                                               vthin, max_up, max_down);
        const bool hfound = find_best<T, false>(p, xyz, range, xyz2, range2, u, v, mul(nh, nh), center, cr, hd, hflip,
                                                hthin, p.search, p.search);
        if ((!vfound && !hfound) || (vthin && hthin)) {  // case A: the beam itself
            n[0] = -beam[0];
            n[1] = -beam[1];
            n[2] = -beam[2];
            break;
        }
        const bool use_v = vfound && (!hfound || hthin);
        const bool use_h = !use_v && hfound && (!vfound || vthin);
        if (use_v || use_h) {  // case B: one neighbour, beam component perpendicular to it
            const double(&one)[3] = use_v ? vd : hd;
            const double denom = dot3(one, one);
            if (fabs(denom) < kEps) break;
            const double sc = dot3(one, beam) / denom;
            const double pr[3] = {sub(beam[0], mul(sc, one[0])), sub(beam[1], mul(sc, one[1])), sub(beam[2], mul(sc, one[2]))};
            const double nsq = dot3(pr, pr);
            if (fabs(nsq) < kEps) break;
            const double len = sqrt(nsq);
            n[0] = -(pr[0] / len);
            n[1] = -(pr[1] / len);
            n[2] = -(pr[2] / len);
            break;
        }
        if (hflip != vflip) {  // case C: cross product of the two neighbour differences
            vd[0] = -vd[0];
            vd[1] = -vd[1];
            vd[2] = -vd[2];
        }
        const double c[3] = {sub(mul(vd[1], hd[2]), mul(vd[2], hd[1])), sub(mul(vd[2], hd[0]), mul(vd[0], hd[2])),
                             sub(mul(vd[0], hd[1]), mul(vd[1], hd[0]))};
        const double mag = sqrt(dot3(c, c));
        if (mag != 0.0) {
            n[0] = c[0] / mag;
            n[1] = c[1] / mag;
            n[2] = c[2] / mag;
        }
    } while (false);
    out[idx * 3 + 0] = static_cast<T>(n[0]);
    out[idx * 3 + 1] = static_cast<T>(n[1]);
    out[idx * 3 + 2] = static_cast<T>(n[2]);
}

}  // namespace

}  // namespace ob

using namespace ob;

extern "C" ob_status ob_normals(ob_dtype dtype, const ob_normals_io* io, ob_stream* s) {
    if (!io || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (dtype != OB_F32 && dtype != OB_F64) return fail(OB_INVALID_ARGUMENT, "unknown dtype");
    // validation order and texts of the reference (normals.cpp:83-88, 418-423, 443-453)
    if (!io->xyz || !io->range || !io->normals) return fail(OB_RUNTIME_ERROR, "normals: xyz dimensions mismatch");
    const bool dual = io->xyz2 != nullptr || io->range2 != nullptr;
    if (dual && (!io->xyz2 || !io->normals2)) return fail(OB_RUNTIME_ERROR, "normals: xyz dimensions mismatch");
    if (dual && !io->range2) return fail(OB_RUNTIME_ERROR, "normals: range2 dimensions mismatch");
    if (io->sensor_origins_xyz && io->n_origins != io->w)
        return fail(OB_RUNTIME_ERROR, "normals: sensor_origins size must match image width");
    if (!(io->target_distance_m > 0.0)) return fail(OB_RUNTIME_ERROR, "normals: target_distance_m must be positive");
    if (!(io->min_angle_of_incidence_rad > 0.0))
        return fail(OB_RUNTIME_ERROR, "normals: min_angle_of_incidence_rad must be positive");
    const size_t F = io->n_frames ? io->n_frames : 1;
    if (io->h == 0 || io->w == 0) return OB_OK;
    if (io->w > 0x7fffffffu || io->h > 0x7fffffffu) return fail(OB_INVALID_ARGUMENT, "frame too large");
    const int device = stream_device(s);
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    const size_t n_px = io->h * io->w, esz = dtype == OB_F64 ? 8 : 4;
    const size_t xyz_fs = io->xyz_frame_stride ? io->xyz_frame_stride : n_px * 3;
    const size_t range_fs = io->range_frame_stride ? io->range_frame_stride : n_px;
    const size_t out_fs = io->normals_frame_stride ? io->normals_frame_stride : n_px * 3;
    Staging stg(st);
    NormalsParams p{};
    // a host output with padding between frames is uploaded first so the padding survives the copy back
    const size_t out_bytes = ((F - 1) * out_fs + n_px * 3) * esz;
    const bool padded = F > 1 && out_fs != n_px * 3;
    auto stage_out = [&](void* host) { return padded ? stg.inout(host, out_bytes) : stg.out(host, out_bytes); };
    p.xyz[0] = stg.in(io->xyz, ((F - 1) * xyz_fs + n_px * 3) * esz);
    p.range[0] = stg.in(io->range, (F - 1) * range_fs + n_px);
    p.out[0] = stage_out(io->normals);
    if (dual) {
        p.xyz[1] = stg.in(io->xyz2, ((F - 1) * xyz_fs + n_px * 3) * esz);
        p.range[1] = stg.in(io->range2, (F - 1) * range_fs + n_px);
        p.out[1] = stage_out(io->normals2);
    }
    if (io->sensor_origins_xyz)
        p.origins = stg.in(io->sensor_origins_xyz, (F - 1) * io->origins_frame_stride + io->w * 3);
    p.subtent[0] = io->vertical_subtent_out ? stg.out(io->vertical_subtent_out, F) : stg.scratch<double>(F);
    if (dual) p.subtent[1] = stg.scratch<double>(F);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage normals buffers");
    p.xyz_fs = xyz_fs;
    p.range_fs = range_fs;
    p.out_fs = out_fs;
    p.origins_fs = io->origins_frame_stride;
    p.H = static_cast<unsigned>(io->h);
    p.W = static_cast<unsigned>(io->w);
    p.n_frames = static_cast<unsigned>(F);
    p.search = static_cast<unsigned>(std::min<size_t>(io->pixel_search_range, 0x7fffffffu));
    p.desired_sq = io->target_distance_m * io->target_distance_m;
    p.tan_safe = std::tan(std::max(io->min_angle_of_incidence_rad, 1e-6));
    p.h_subtent = 2.0 * M_PI / static_cast<double>(io->w);
    p.subtent_override = io->vertical_subtent_rad;
    p.dual = dual ? 1 : 0;
    if (F > 65535) return fail(OB_INVALID_ARGUMENT, "too many frames in one call");
    const dim3 grid((p.W + 31) / 32, (p.H + 7) / 8, static_cast<unsigned>(F));
    if (grid.y > 65535) return fail(OB_INVALID_ARGUMENT, "frame too tall");
    const unsigned sub_threads = dual ? 64 : 32;  // one warp per return
    if (dtype == OB_F64) {
        launch(OB_FAM_NORMALS, normals_subtent_kernel<double>, static_cast<unsigned>(F), sub_threads, 0, st, p);
        launch(OB_FAM_NORMALS, normals_kernel<double>, grid, 256, 0, st, p, 0);
        if (dual) launch(OB_FAM_NORMALS, normals_kernel<double>, grid, 256, 0, st, p, 1);
    } else {
        launch(OB_FAM_NORMALS, normals_subtent_kernel<float>, static_cast<unsigned>(F), sub_threads, 0, st, p);
        launch(OB_FAM_NORMALS, normals_kernel<float>, grid, 256, 0, st, p, 0);
        if (dual) launch(OB_FAM_NORMALS, normals_kernel<float>, grid, 256, 0, st, p, 1);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "normals launch");
    e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "normals D2H");
    return OB_OK;
}
