// ob_internal.h -- internal declarations shared by the kernels and the C-ABI glue.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <string>
#include <utility>

#include "../../include/ouster_b200.h"

namespace ob {

constexpr int kMaxRows = 512;  // rows (beams) whose shifts travel as kernel parameters

struct Tunables {
    int cloud_tw;          // pixels per tile (multiple of 4)
    int cloud_stages;      // TMA ring depth
    int cloud_threads;     // threads per CTA
    int cloud_ctas_per_sm; // persistent CTAs per SM
    int cloud_pose_tw;     // pixels per row of a tile of the pose-fused variant
    int cloud_pose_stages, cloud_pose_ctas_per_sm;
    int cloud_pose_threads;  // compute threads per CTA of the pose-fused variant
    int cloud_pose_rows;   // rows per work item of the pose-fused variant (one pose slice load per item)
    int cloud_store_lag;   // 1: refill the stage of tile k-2 instead of k-1 (hides the store drain)
    int cloud_auto;        // 1: nobody touched the cloud_* geometry -> launch_cloud picks it per return count
    int decode_stages;
    int decode_threads;
    int decode_ctas_per_sm;
    int decode_tile_packets;  // packets (groups of columns_per_packet columns) per tile
    int decode_runtime_plans; // 1: never use the compile-time pixel layouts (testing / comparison)
    int decode_prefetch;      // L2 prefetch of the next tile: 0 off, 1 at tile start (evict_last), 2 before phase B
    int decode_pipe;          // 1 (default): pipelined K2 (ob_decode_pipe.cu) whenever the launch is eligible
    int decode_pipe_warps;    // compute warps of the pipelined K2 (24)
    int decode_pipe_dyn_rows; // phase A rows of the pipelined K2: 0 fixed stride, 1 all through a counter, 2 last round through a counter, 3 (default) 1 with a fused cloud else 0
    int decode_pipe_tma_xyz;      // phase B of the pipelined K2 leaves XYZ in the LUT slot and a store warp writes it out with tensor copies (dual return, uniformly strided batch); default 0
    int decode_pipe_ctas;         // CTAs per SM of the pipelined K2: 1, 2..4 (the warps split between them, 64-register build), 0 = auto (2 where the stages fit)
    int decode_pipe_helpers;      // extra phase-A-only warps of the pipelined K2 (0..6; > 0 selects the 64-register build)
    int decode_pipe_lane_arrive;  // 1 (default): per-lane arrivals on the stage-free barrier (racecheck-clean)
    int decode_pipe_pk_split;  // bulk copies per packet (more TMA operations in flight per SM)
    int decode_pipe_lut_split; // tensor copies per table and LUT sub-tile
    int decode_pipe_prefetch; // L2 prefetch distance (tiles) of the pipelined K2's packet loads, 0 = off
    int force_generic;     // 1: K1 takes the generic GPU kernel (any width / alignment) instead of the TMA one
    int sm_count;
};
const Tunables& tunables(int device);
bool set_tunable(int device, const char* name, int value);

// LUT-free ("analytic") projection of a LUT built from per-beam intrinsics (ouster_core/src/xyzlut.cpp:35-86
// refactored): direction = R * (cos(enc+az)cos(alt), sin(enc+az)cos(alt), sin(alt)), offset from the same
// angles, so XYZ = M * ((r - dist) * d_beam + (cos(enc) b03, sin(enc) b03, b23)) with M = [R|t] * range_unit.
// Per-row and per-column tables replace the 24 B/pixel LUT stream.  Lives in device memory.
template <typename T>
struct LutAnalyticT {
    const T* row;  // H x 4: cos(az)cos(alt), sin(az)cos(alt), sin(alt), 0
    const T* col;  // W x 2: cos(enc), sin(enc)
    T dist, b03, b23;
    T m[12];       // row-major 3x4, already scaled by range_unit
};

// ---- launchers implemented in the .cu files; all return cudaError_t ----
template <typename T>
struct CloudArgs {
    const T* dir;
    const T* off;
    const uint32_t* range;
    T* xyz;
    uint32_t* rd;
    T* xd;
    size_t range_fs, range_rs, xyz_fs, xyz_rs, rd_fs, rd_rs, xd_fs, xd_rs;
    int H, W, n_returns;
    uint32_t n_frames;
    const uint16_t* shift;  // H entries, already reduced to [0, W) (host memory); may be null if no rd/xd
    const T* poses{nullptr};  // optional per-column poses: n_frames x W x 16 (device), fused dewarp
    size_t poses_fs{0};
    const LutAnalyticT<T>* analytic{nullptr};  // device; non-null: recompute direction/offset, dir/off unused
};

template <typename T>
cudaError_t launch_cloud(const CloudArgs<T>& a, int device, cudaStream_t st);

template <typename T>
cudaError_t launch_dewarp(const T* pts, const T* poses, T* out, size_t H, size_t W, cudaStream_t st);

cudaError_t launch_destagger(size_t elem_size, size_t k, const void* img, const uint16_t* shift_host,
                             size_t h, size_t w, void* out, int device, cudaStream_t st);

cudaError_t launch_make_lut(size_t w, size_t h, double range_unit, const double* b2l16,
                            const double* tr16, const double* az_dev, size_t n_az,
                            const double* alt_dev, size_t n_alt, double* dir_dev, double* off_dev,
                            cudaStream_t st);
cudaError_t launch_cast_f64_f32(const double* src, float* dst, size_t n, cudaStream_t st);

// ---- K3: range -> posed, filtered, compacted point list, one launch (ob_dewarp_frame.cu) ----
// one entry per frame of the launch (a single frame or the frames of a FrameSet), device memory
struct K3Frame {
    const uint32_t* range;       // H x W
    const void* dir;             // LUT tables of the launch's dtype
    const void* off;
    const double* poses;         // W x 16
    const uint32_t* status;      // W
    const uint64_t* timestamps;  // W, nullable
    unsigned H, W, n_cg, n_slabs;  // n_cg = ceil(W / 32) CTAs, n_slabs = ceil(H / 16)
    unsigned first_block;        // logical index of the frame's first CTA (sum of n_cg of the frames before)
    unsigned index;              // the frame's index in the set (reported as frame_idx)
};
// tallest frame K3 takes: a CTA keeps one count per (16-row slab, column) for its 32 columns in shared memory, and
// 1600 slabs of them are 200 KB
constexpr size_t kDewarpMaxRows = 25600;
size_t dewarp_scan_scratch_bytes(unsigned n_blocks, unsigned n_frames);
// *frame_end_dev: device array [n_frames], points up to and including frame f (valid when the launch is done)
cudaError_t launch_dewarp_fused(const K3Frame* frames_dev, unsigned n_frames, unsigned n_blocks, unsigned max_slabs,
                                uint32_t min_r, uint32_t max_r, int dtype, void* scratch, void* points,
                                uint32_t* frame_idx, uint32_t* col_idx, uint64_t* ts_out, unsigned long long capacity,
                                const unsigned long long** frame_end_dev, cudaStream_t st);

// ---- decode ----
struct DecodeField {  // device-side copy of ob_field_desc, pre-digested
    uint32_t offset;
    uint32_t elem_size;
    uint64_t mask;
    int32_t shift;
    int32_t range_return;
    uint32_t zero_pattern;
    uint32_t pad;
};

struct DecodeLayout {
    uint32_t packet_header_size, col_header_size, channel_data_size, col_size, packet_size;
    uint32_t cpp, H, W;
    DecodeField ts, mid, status;
    uint32_t n_fields;
    DecodeField fields[OB_MAX_FIELDS];
};

// DecodeFrame::flags
constexpr uint32_t kFrameIdentityMap = 1u;  // col_src is null: column j comes from slot j / cpp, column j % cpp
constexpr uint32_t kFrameBulkPackets = 2u;  // packets, packet_stride and packet_size are 16-byte aligned
constexpr uint32_t kFrameAllFields = 4u;    // every decoder field has an output image

struct DecodeFrame {  // one per frame of a batched launch, lives in device memory
    const uint8_t* packets;
    unsigned long long packet_stride;
    uint32_t n_slots;
    uint32_t flags;          // kFrame* bits
    const int32_t* col_src;  // device, W entries (unused when identity)
    void* fields[OB_MAX_FIELDS];
    uint64_t* timestamp;
    uint16_t* measurement_id;
    uint32_t* status;
    void* xyz[OB_MAX_RETURNS];
    uint32_t* rd[OB_MAX_RETURNS];
    const void* lut_dir;  // per-frame LUT (independent sensor streams in one launch); null: launch-level
    const void* lut_off;
    const void* lut_maps;  // device copy of the LUT's two TMA descriptors (direction, offset) or null
    const void* lut_an;    // device LutAnalyticT<T> of the frame's LUT when its LUT-free mode is on, else null
};

struct DecodeLaunch {
    const DecodeLayout* layout_host;  // travels as a kernel parameter
    const DecodeFrame* frames_dev;
    uint32_t n_frames;
    const void* lut_dir;  // nullable
    const void* lut_off;
    int lut_dtype;
    const uint16_t* shift_host;  // nullable (H entries reduced to [0,W))
    bool vec_ok;                 // LUT / XYZ pointers are 16-byte aligned
    const void* lut_maps{nullptr};  // TMA descriptors of the launch-level LUT (lut_tensor_maps) or null
    const void* lut_an{nullptr};    // launch-level LUT in LUT-free mode: device LutAnalyticT<T>
    bool frame_luts_have_maps{true};  // every per-frame LUT of the table carries lut_maps
    // XYZ outputs of a uniformly strided batch (frame f at base + f * stride): lets the pipelined kernel store
    // them with tensor copies; null when the frames' XYZ pointers are unrelated
    const void* xyz_base[2]{nullptr, nullptr};
    unsigned long long xyz_frame_stride{0};
    bool any_xyz{true};          // some frame of the launch asks for the fused cloud (tuning hint only)
};
cudaError_t launch_decode(const DecodeLaunch& a, int device, cudaStream_t st);

// ---- pipelined K2 (ob_decode_pipe.cu) ----
struct DecodeParams;
// TMA box (in LUT scalars x rows) the pipelined kernel would use for this decoder, false if it cannot run
bool decode_pipe_box(const DecodeLayout& L, int device, int lut_dtype, uint32_t* box_w, uint32_t* box_h);
// device pointer to two CUtensorMap (direction, offset) describing `box_w x box_h` tiles of a LUT, created
// on first use and cached; null when the driver entry point is unavailable or the LUT is not 16-byte aligned
const void* lut_tensor_maps(const void* dir, const void* off, int dtype, size_t h, size_t w, uint32_t box_w,
                            uint32_t box_h, int device);
void forget_lut_tensor_maps(const void* dir);
// packets per tile, compute warps per CTA and CTAs per SM of the pipelined kernel for this layout
void decode_pipe_shape(const DecodeLayout& L, int device, uint32_t* P, uint32_t* ncw, uint32_t* ctas);
bool decode_pipe_eligible(const DecodeParams& p, const DecodeLaunch& a, int device);
cudaError_t launch_decode_pipe(DecodeParams& p, const DecodeLaunch& a, int device, cudaStream_t st);
cudaError_t make_decode_params(const DecodeLaunch& a, int device, bool pipe, DecodeParams& p);

// Kernel families of ob_kernel_launch_count_of; the names are in ob_api.cu.  DECODE_PIPE is a sub-family of
// DECODE: a launch counted as DECODE_PIPE also counts as DECODE, and ob_kernel_launch_count leaves it out.
enum { OB_FAM_DECODE_PIPE = 0, OB_FAM_DECODE = 1, OB_FAM_CLOUD = 2, OB_FAM_NORMALS = 3, OB_FAM_VOXEL = 4,
       OB_FAM_VOXEL_MAP = 5, OB_FAM_ICP = 6, OB_FAM_ALIGN = 7, OB_FAM_ZONE = 8, OB_FAM_IMAGE = 9,
       OB_FAM_FRAME_OPS = 10, OB_FAM_POSE = 11, OB_FAM_DEWARP = 12, OB_FAM_DESTAGGER = 13, OB_FAM_LUT = 14,
       OB_FAM_ENCODE = 15, OB_FAM_GROUND = 16, OB_FAM_COUNT = 17 };
void record_launch(int family);

// Every kernel of the library is launched through here, so the launch counters cannot drift from the launches.
// Errors are left to the caller's cudaGetLastError().  The kernels CUB launches inside DeviceRadixSort and
// DeviceScan do not come through here and are not counted.
template <typename... P, typename... A>
void launch(int family, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
    kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    record_launch(family);
}

}  // namespace ob
