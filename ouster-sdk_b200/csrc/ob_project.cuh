// ob_project.cuh -- the per-pixel arithmetic of range -> XYZ and of the per-column pose, shared by K1 and the
// stand-alone dewarp (ob_cloud.cu), K3 (ob_dewarp_frame.cu), the map-row ingest (ob_map_rows.cu), the frame
// operations (ob_frame_ops.cu) and ground segmentation (ob_ground.cu), so that every path rounds exactly alike.
#pragma once
#include <cstdint>

namespace ob {

// r * dir + ofs with the int->float conversion and two roundings of the reference loop
// (impl::cartesianT, impl/cartesian.h:36-66); range 0 gives 0
__device__ __forceinline__ float project(uint32_t r, float d, float o) {
    return r == 0 ? 0.0f : __fadd_rn(__fmul_rn(static_cast<float>(r), d), o);
}
__device__ __forceinline__ double project(uint32_t r, double d, double o) {
    return r == 0 ? 0.0 : __dadd_rn(__dmul_rn(static_cast<double>(r), d), o);
}

// pose of one column applied to one point: R*p + t with every product rounded on its own and the
// sum taken as x0 + (x1 + x2), then + t (pose_util.h:37-59; same helper as the stand-alone dewarp)
__device__ __forceinline__ float pose_row(const float* m, float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fadd_rn(__fmul_rn(m[1], y), __fmul_rn(m[2], z))), m[3]);
}
__device__ __forceinline__ double pose_row(const double* m, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dadd_rn(__dmul_rn(m[1], y), __dmul_rn(m[2], z))), m[3]);
}

}  // namespace ob
