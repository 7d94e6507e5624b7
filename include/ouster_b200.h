/*
 * ouster_b200.h -- C ABI of the CUDA scan->pointcloud path (H100, sm_90a).
 *
 * Drop-in boundary for the hot path of ouster_core (ouster-sdk 1.0.1):
 *   packet field decode (PacketFormat) -> LidarFrame/LidarScan -> destagger() -> XYZLut/cartesian().
 * The reference reaches this path through C++ symbols in namespace ouster::sdk::core (there is
 * no plugin ABI, SURVEY 8b); the replacement headers under include/ouster/core/ keep those C++
 * signatures and call the entry points below.  Each entry point cites the reference interface
 * it replaces (paths relative to the reference tree).
 *
 * Conventions
 *  - every function returns an ob_status; on failure ob_last_error() holds the exact message text
 *    of the exception the reference would have thrown (thread-local).  No exception crosses the ABI.
 *  - every data pointer may be device memory, pinned host memory or pageable host memory; the kind
 *    is detected with cudaPointerGetAttributes.  Host buffers are staged through the ob_stream's
 *    device arena (H2D before the kernel, D2H after it, all on the stream).
 *  - calls are asynchronous on the ob_stream; ob_stream_sync() makes host-visible results final.
 *  - handles (ob_lut, ob_decoder) are immutable after creation and may be shared by threads;
 *    an ob_stream belongs to one caller thread at a time (one per sensor stream, like FrameBatcher).
 *  - there is NO CPU fallback: without a CUDA device every compute call fails with OB_NO_DEVICE.
 */
#ifndef OUSTER_B200_H
#define OUSTER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OB_ABI_VERSION 1
#define OB_MAX_FIELDS 24  /* decoded channel fields per packet format */
#define OB_MAX_RETURNS 2

typedef enum ob_status {
    OB_OK = 0,
    OB_INVALID_ARGUMENT = 1, /* std::invalid_argument in the reference */
    OB_RUNTIME_ERROR = 2,    /* std::runtime_error in the reference */
    OB_CUDA_ERROR = 3,
    OB_NO_DEVICE = 4
} ob_status;

typedef enum ob_dtype { OB_F32 = 0, OB_F64 = 1 } ob_dtype;

/* Handles (ob_stream, ob_lut, ob_decoder, ob_decode_job, ob_voxel_map, ob_zone_monitor, ob_image_proc) live on the
 * device they were created for.  Every *_destroy frees the handle's memory on that device and leaves the caller's
 * current device as it was, so a handle may be destroyed from anywhere (a garbage collector, another device's code).
 * Passing NULL to a *_destroy is OB_OK. */
typedef struct ob_stream ob_stream;   /* CUDA stream + device arena + pinned staging */
typedef struct ob_lut ob_lut;         /* device-resident XYZLutT<T> (direction/offset tables) */
typedef struct ob_decoder ob_decoder; /* device-resident PacketFormat decode table */

/* ---- library ---- */
int ob_abi_version(void);
/* sizeof() of a public struct by name ("ob_cloud_io", "ob_field_desc", "ob_packet_layout",
 * "ob_decode_io", "ob_decode_batch", "ob_dewarp_frame_io", "ob_normals_io", "ob_encode_io", "ob_dewarp_frames_io",
 * "ob_voxel_io", "ob_point_rows", "ob_voxel_map_cull_io", "ob_voxel_query_io", "ob_icp_io", "ob_icp_system_io",
 * "ob_cloud_align_io", "ob_cloud_nearest_io", "ob_zone_desc", "ob_zone_render_io", "ob_zone_live", "ob_zone_state",
 * "ob_image_params", "ob_image_state", "ob_frame_field", "ob_frame_ops_io", "ob_frame_rows_entry",
 * "ob_frame_rows_io", "ob_map_rows", "ob_map_field", "ob_map_rows_item", "ob_interp_pose_io",
 * "ob_frame_poses_item", "ob_ground_model", "ob_ground_item", "ob_align_clouds_trace", "ob_align_clouds_io");
 * 0 for unknown names.  Lets FFI bindings verify their layout. */
size_t ob_abi_sizeof(const char* struct_name);
const char* ob_last_error(void);
/* number of visible CUDA devices (0 without a driver/GPU); never fails */
int ob_device_count(void);
/* kernels launched by this library since load (all threads), not counting those CUB launches inside its
 * sorts and scans; the sum of the families below except "decode_pipe".  The bench's gpu_launches claim */
uint64_t ob_kernel_launch_count(void);
/* launches of one named kernel family since load: "decode_pipe" (pipelined K2, also counted in "decode"),
 * "decode" (K2, any kernel), "cloud" (K1), "normals", "voxel", "voxel_map", "icp", "align", "zone", "image",
 * "frame_ops", "pose", "dewarp" (K3 and the per-column dewarp), "destagger", "lut" (LUT from intrinsics and
 * its f32 cast), "encode" (K4), "ground"; 0 for unknown names.  Every launch belongs to exactly one family, so tests
 * can assert which code path ran. */
uint64_t ob_kernel_launch_count_of(const char* name);
/* tuning hook (launch geometry and code-path selection only, never results): cloud_tw, cloud_stages,
 * cloud_threads (compute threads; a copy warp is added), cloud_ctas_per_sm, cloud_store_lag,
 * cloud_pose_tw, cloud_pose_stages, cloud_pose_ctas_per_sm, decode_stages, decode_threads,
 * decode_ctas_per_sm, decode_tile_packets, decode_prefetch, decode_runtime_plans, force_generic (K1: generic GPU kernel
 * instead of the TMA one), cloud_auto (1: K1 picks its geometry per launch, e.g. wider tiles for single-return float
 * frames; setting cloud_tw, cloud_stages, cloud_threads or cloud_ctas_per_sm clears it, setting it to 1 restores
 * the automatic choice).
 * Defaults come from OB_* environment variables of the same (upper-case) names; cloud_auto starts at 0 when one of
 * OB_CLOUD_TW, OB_CLOUD_STAGES, OB_CLOUD_THREADS or OB_CLOUD_CTAS_PER_SM is set, else at 1. */
ob_status ob_set_tunable(int device, const char* name, int value);

/* ---- streams ---- */
ob_status ob_stream_create(int device, ob_stream** out);
/* wrap a caller-owned cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream) */
ob_status ob_stream_wrap(int device, void* cuda_stream, ob_stream** out);
ob_status ob_stream_sync(ob_stream* s);
void* ob_stream_cuda_handle(ob_stream* s);
ob_status ob_stream_destroy(ob_stream* s);

/* pinned host allocations for callers that want full-rate H2D/D2H */
ob_status ob_host_alloc(size_t bytes, void** out);
ob_status ob_host_free(void* p);

/* ---- XYZ lookup table ----
 * replaces XYZLutT<T>(direction, offset, h, w)            ouster_core/include/ouster/core/xyzlut.h:135
 *          impl::make_xyz_lut(w,h,range_unit,b2l,tf,az,alt) ouster_core/src/xyzlut.cpp:11-89
 * direction/offset: row-major (h*w) x 3 of dtype (ArrayX3R<T>, typedefs.h:71).
 * ob_lut_from_intrinsics builds the table on the GPU in double and casts to dtype (xyzlut.h:119-124).
 * errors: "lut dimensions must be greater than zero", "unexpected frame dimensions" (xyzlut.cpp:15,20)
 */
ob_status ob_lut_create(ob_dtype dtype, const void* direction, const void* offset, size_t h,
                        size_t w, int device, ob_lut** out);
ob_status ob_lut_from_intrinsics(ob_dtype dtype, size_t w, size_t h, double range_unit,
                                 const double* beam_to_lidar_transform /* 4x4 row-major */,
                                 const double* transform /* 4x4 row-major */,
                                 const double* azimuth_angles_deg, size_t n_azimuth,
                                 const double* altitude_angles_deg, size_t n_altitude, int device,
                                 ob_lut** out);
/* copy the tables back to host arrays of the LUT's dtype (XYZLutT::direction / ::offset members) */
ob_status ob_lut_download(const ob_lut* lut, void* direction, void* offset);
ob_status ob_lut_info(const ob_lut* lut, size_t* h, size_t* w, int* dtype, int* device);
/* device pointers of the tables (for zero-copy consumers such as torch tensors) */
ob_status ob_lut_device_ptrs(const ob_lut* lut, void** direction, void** offset);
/* LUT-free projection (opt-in, SURVEY 8d): a lut made by ob_lut_from_intrinsics from per-beam angles
 * (n_azimuth == n_altitude == h) can have its direction/offset recomputed inside the kernels from
 * per-row (cos az cos alt, sin az cos alt, sin alt) and per-column (cos enc, sin enc) tables and the
 * 3x4 extrinsic -- the factorisation of ouster_core/src/xyzlut.cpp:35-86 -- instead of streaming
 * 24 B/pixel of LUT.  Results agree with the LUT path to <= 1e-5 norm-wise relative (float
 * rounding), NOT bit for bit, which is why it is off by default.  Set it before the handle is shared
 * between threads.  error: "LUT-free projection needs a lut built from per-beam intrinsics". */
ob_status ob_lut_set_analytic(ob_lut* lut, int enable);
int ob_lut_is_analytic(const ob_lut* lut);
ob_status ob_lut_destroy(ob_lut* lut);

/* ---- range -> XYZ ----
 * replaces XYZLutT<T>::operator()(range)     xyzlut.h:139-143
 *          impl::cartesianT<T>(points, ...)   ouster_core/include/ouster/core/impl/cartesian.h:36-66
 *          cartesian(range, lut)              ouster_core/src/xyzlut.cpp:116-124
 * range: n_pixels uint32 (staggered H x W), xyz: n_pixels x 3 of the LUT dtype.
 * error: "unexpected image dimensions" when n_pixels != h*w (xyzlut.cpp:117-119)
 */
ob_status ob_cartesian(const ob_lut* lut, const uint32_t* range, size_t n_pixels, void* xyz,
                       ob_stream* s);

/* ---- destagger / stagger ----
 * replaces destagger_into<T>/destagger<T>/stagger<T> (2-D and N-D forms)
 *          ouster_core/include/ouster/core/impl/lidar_frame_impl.h:733-811, 825-989
 * img/out: row-major h x w x k elements of elem_size bytes (k = product of trailing dims, 1 for 2-D).
 * d[u][j] = g[u][(j - s_u) mod w]; inverse negates s_u.
 * errors: "image height does not match shifts size" (:741)
 */
ob_status ob_destagger(size_t elem_size, size_t k, const void* img, const int32_t* pixel_shift_by_row,
                       size_t n_shifts, size_t h, size_t w, int inverse, void* out, ob_stream* s);

/* ---- per-column pose application (SURVEY 8f #1) ----
 * replaces dewarp<T>(dewarped, points, poses)   ouster_core/include/ouster/core/pose_util.h:37-59
 *          transform<T>(transformed, points, pose)  pose_util.h:118-131  (n_poses == 1)
 * points/out: n_points x 3 of dtype, row-major, point i*n_poses + w uses pose w;
 * poses: n_poses x 16 of dtype (row-major 4x4 each).  n_points must be a multiple of n_poses.
 */
ob_status ob_dewarp(ob_dtype dtype, const void* points, const void* poses, size_t n_points,
                    size_t n_poses, void* out, ob_stream* s);

/* ---- pose interpolation (DESIGN f-12) ----
 * replaces core::interp_pose(x_interp, t0, x0, t1, x1)      ouster_core/include/ouster/core/pose_util.h:316-326
 *          core::interp_pose(x_interp, x_known, poses_known) and the MatrixX16R<float | double> overload
 *                                                            pose_util.h:360-434 (impl::interp_pose, :243-286)
 *          python interp_pose / interp_pose_float            python/src/cpp/client/processing.cpp:241-338
 * Between knots k[i] < k[i+1] the pose at x is a * exp((x - k[i]) * (1 / (k[i+1] - k[i])) * log(a^-1 b)), a and b
 * the knots' poses; x is split into segments by the reference's lower_bound walk on any input, the part after the
 * last knot takes the last segment, and x - k[i] is taken in the x dtype before it is widened.
 * x_interp, x_known: float64 or int64 (x_dtype); poses_known m x 16 and poses n x 16 of pose_dtype (row-major 4x4):
 * OB_F64 is interp_pose, OB_F32 is interp_pose_float (the known poses are widened, each result rounded once).
 * two_pose = 1: interp_pose(x, t0, x0, t1, x1) with x_known = {t0, t1} (m == 2): no knot-order check, and the zero
 * duration check runs even for n == 0.
 * Errors, OB_INVALID_ARGUMENT with the reference's texts, in the reference's order: "Not enough evaluation poses for
 * interpolation" (m < 2, on the host), then as the walk meets them "input x_known values are not monotonically
 * increasing or values repeated", "Cannot interpolate with zero duration between poses" (|t1 - t0| < epsilon of the x
 * dtype: never for int64) and "x_interp values must be monotonically increasing: <x[j]> < <x[j-1]>" (std::to_string).
 * NaN compares false, so it never fails a check.  A failing call writes no pose.
 * error == NULL: the call waits for the check and fails with the text; with host outputs it waits again for them.
 * error = 3 int64 in DEVICE memory (poses must then be device memory too): nothing waits, the words (kind
 * ob_pose_error, index, 0) are written in stream order and the call can be captured in a CUDA graph.
 * Launches (family "pose"): three, one when n == 0.  Pointers may be host or device memory. */
typedef enum ob_pose_x_dtype { OB_POSE_X_F64 = 0, OB_POSE_X_I64 = 1 } ob_pose_x_dtype;
typedef enum ob_pose_error {
    OB_POSE_OK = 0,
    OB_POSE_KNOT_ORDER = 1,    /* index: i, with x_known[i] >= x_known[i + 1] */
    OB_POSE_ZERO_DURATION = 2, /* index: the segment */
    OB_POSE_DESCENT = 3        /* index: j, with x[j] < x[j - 1] (in ob_frames_interp_pose: the column) */
} ob_pose_error;
typedef struct ob_interp_pose_io {
    const void* x_interp; /* n values of x_dtype */
    size_t n;
    const void* x_known;  /* m values of x_dtype */
    size_t m;
    int x_dtype;          /* ob_pose_x_dtype */
    int pose_dtype;       /* ob_dtype */
    int two_pose;
    int pad;
    const void* poses_known; /* m x 16 */
    void* poses;             /* n x 16 */
    int64_t* error;          /* NULL, or 3 words of device memory */
} ob_interp_pose_io;
ob_status ob_interp_pose(const ob_interp_pose_io* io, ob_stream* s);

/* replaces mapping::ConstantVelocityDeskewMethod::update over a FrameSet     ouster_mapping/src/deskew_method.cpp:55-71
 *          mapping::impl::interp_pose(frame, t0, x0, t1, x1)                 deskew_method.cpp:29-37
 *          impl::init_valid_column_poses(frame_set, pose)  (x1 == NULL)      ouster_mapping/src/slam_util.cpp:129-140
 * For every frame of the set in slot order (timestamps == NULL marks an empty slot): the valid columns
 * (status & 1) get the pose at double(timestamp) * 1e-9 between (t0, x0) and (t1, x1); other columns keep their
 * bytes.  x1 == NULL: every valid column gets x0.  x0 / x1: 16 doubles, host or device memory (e.g. a device pose of
 * ob_icp_align).  Errors in the reference's order: "Cannot interpolate with zero duration between poses" is known
 * on the host and fails the call before anything runs when the set has a frame; a decreasing valid timestamp in a
 * frame fails "x_interp values must be monotonically increasing: ..." with the frames before it written and that
 * frame and the later ones untouched.  error: as for ob_interp_pose (kind, column, slot); host poses are fine with
 * it, since every frame's poses are copied in and out whole.
 * Launches (family "pose"): two (a check block per frame, then the write), one with x1 == NULL, none for a set
 * without columns.  Buffers may be host or device memory.
 * CUDA graphs: with device buffers and a device error word the call can be captured once it has run on the stream
 * with the same frames.  The frame table lives in the ob_stream and is rewritten in place by the next call on that
 * stream with a different set, so a graph captured earlier then reads that set: after such a call, capture the
 * graph again (or give each graph its own ob_stream). */
typedef struct ob_frame_poses_item {
    const uint64_t* timestamps; /* w: LidarFrame::timestamp; NULL: empty slot */
    const uint32_t* status;     /* w: LidarFrame::status */
    double* poses;              /* w x 16: LidarFrame::body_to_world */
    size_t w;
} ob_frame_poses_item;
ob_status ob_frames_interp_pose(const ob_frame_poses_item* frames, size_t n_frames, double t0, const double* x0,
                                double t1, const double* x1, int64_t* error, ob_stream* s);

/* ---- range image -> world-frame point list (projection + pose + range filter + compaction) ----
 * replaces dewarp<T>(const LidarFrame&, const XYZLutT<T>&, min_range, max_range)
 *                                                ouster_core/include/ouster/core/pose_util.h:456-485
 *          impl::dewarp_impl (single frame)      ouster_core/include/ouster/core/impl/dewarp_impl.h:22-76
 * Columns between the first and the last column with status bit 0 set are visited in order, columns
 * whose status word is 0 are skipped, and inside a column the pixels with
 * ceil(min_range*1e3) <= r <= floor(max_range*1e3) are emitted top to bottom as R_col*lut(r) + t_col
 * (body_to_world cast to the LUT dtype) -- the reference's order and arithmetic, without
 * materialising the full cloud first (the fusion its own note at dewarp_impl.h:27-29 asks for).
 * Range window: ceil(min_range*1e3) and floor(max_range*1e3) are computed in double, as the reference does, and
 * must both be finite and in [0, 4294967295] (a ceil of -0.0 counts as 0); otherwise the call fails with
 * OB_INVALID_ARGUMENT before anything is staged, since the reference's conversion of such a bound to uint32 is
 * undefined.  To keep every range, pass max_range = 4294967.295.  A minimum above the maximum is a valid, empty
 * window (nothing is launched).  Frames may have at most 25600 rows (a taller one fails with OB_INVALID_ARGUMENT
 * before anything is staged).
 * ONE kernel launch (count, decoupled look-back scan and emit fused; the count is a device-side word).
 * n_points in host memory: the call waits for the count and, when outputs are in host memory, then for their
 * points (host outputs are final on return, device outputs after ob_stream_sync); it raises
 * "output capacity too small" when more than `capacity` points pass the filter, with *n_points left 0 and the
 * host outputs untouched.
 * n_points in DEVICE memory (8 bytes; all outputs in device memory): nothing waits for the GPU, the count is
 * written in stream order next to the points, and a count above `capacity` means the list was cut there.  A host
 * output with a device n_points is refused before anything is launched, with the count 0.
 */
typedef struct ob_dewarp_frame_io {
    const uint32_t* range;       /* h x w, staggered (the RANGE field) */
    const double* poses;         /* w x 16: LidarFrame::body_to_world (row-major 4x4 per column) */
    const uint32_t* status;      /* w: LidarFrame::status */
    const uint64_t* timestamps;  /* w: LidarFrame::timestamp; only read when timestamps_out != NULL */
    double min_range, max_range; /* metres */
    void* points;                /* capacity x 3 of the LUT dtype */
    uint32_t* col_idx;           /* optional: column of every point */
    uint64_t* timestamps_out;    /* optional: column timestamp of every point */
    size_t capacity;             /* in points; h*w always suffices */
} ob_dewarp_frame_io;
ob_status ob_dewarp_frame(const ob_lut* lut, const ob_dewarp_frame_io* io, size_t* n_points, ob_stream* s);

/* ---- the frames of a set in one go ----
 * replaces dewarp<T>(const FrameSet&, const std::vector<XYZLutT<T>>&, min_range, max_range)
 *                                                ouster_core/include/ouster/core/pose_util.h:475
 *          impl::dewarp_impl (FrameSet)          ouster_core/include/ouster/core/impl/dewarp_impl.h:84-117
 * Every frame has its own LUT (lut == NULL marks an empty slot of the set, skipped like
 * FrameSet::valid_indices()), range image, poses, status and timestamps; the points of frame i follow those
 * of the frames before it, each frame in the single-frame order above.  ONE launch for the whole set (the
 * look-back chain of the compaction simply continues across the frames); n_points may be device memory as
 * for ob_dewarp_frame (then counts must be NULL).
 * Optional per-point provenance: frame index, column index, column timestamp (dewarp_impl.h:88-90).
 * counts[i] (optional, n_frames entries, host memory) = points of slot i; zeroed on entry and filled only by a
 * call that succeeds.
 * Buffers may be host or device memory.  The range window and row limit are those of ob_dewarp_frame.
 * errors: "output capacity too small", "the luts of a set must share one dtype". */
typedef struct ob_dewarp_frames_io {
    const ob_lut* lut;           /* NULL: no frame in this slot */
    const uint32_t* range;       /* h x w, staggered */
    const double* poses;         /* w x 16 */
    const uint32_t* status;      /* w */
    const uint64_t* timestamps;  /* w; only read when timestamps_out != NULL */
} ob_dewarp_frames_io;
ob_status ob_dewarp_frames(const ob_dewarp_frames_io* frames, size_t n_frames, double min_range, double max_range,
                           void* points, size_t capacity, uint32_t* frame_idx, uint32_t* col_idx,
                           uint64_t* timestamps_out, size_t* counts, size_t* n_points, ob_stream* s);

/* ---- surface normals on destaggered XYZ (SURVEY 8f-2) ----
 * replaces algorithm::normals(xyz, range, sensor_origins_xyz, pixel_search_range, min_angle_of_incidence_rad,
 *          target_distance_m) and the dual-return overload
 *                                ouster_algorithm/include/ouster/algorithm/normals.h:58-108
 *          compute_unit_normals / compute_vertical_subtent   ouster_algorithm/src/normals.cpp:32-407
 * Inputs are DESTAGGERED images (e.g. ob_cloud_io.xyz_destaggered / range_destaggered, in place on the
 * device); xyz2/range2/normals2 all set = the dual-return overload (the returns see each other's points
 * as neighbours; the second return's pass uses the first return's vertical pixel subtent when that is
 * > 0, and otherwise derives its own from xyz2/range2, as compute_unit_normals ignores an override of 0).
 * dtype = scalar type of
 * xyz* and normals* (the reference is double; float inputs are widened, results rounded once).
 * n_frames > 1 batches independent frames (strides in ELEMENTS, 0 = dense).
 * errors (OB_RUNTIME_ERROR, the reference's std::runtime_error texts): "normals: target_distance_m
 * must be positive", "normals: min_angle_of_incidence_rad must be positive", "normals: sensor_origins
 * size must match image width", "normals: xyz dimensions mismatch", "normals: range2 dimensions mismatch".
 */
typedef struct ob_normals_io {
    size_t n_frames; /* 0 or 1: a single frame */
    size_t h, w;
    const void* xyz;              /* h*w x 3 */
    const uint32_t* range;        /* h x w */
    const void* xyz2;             /* optional second return */
    const uint32_t* range2;
    void* normals;                /* h*w x 3 */
    void* normals2;
    size_t xyz_frame_stride, range_frame_stride, normals_frame_stride;
    const double* sensor_origins_xyz; /* n_origins x 3 per-column sensor origins, NULL = zeros */
    size_t n_origins;                 /* must equal w when sensor_origins_xyz is set */
    size_t origins_frame_stride;      /* in doubles; 0 = the same origins for every frame */
    size_t pixel_search_range;        /* reference default 1 */
    double min_angle_of_incidence_rad; /* reference default 1 deg (normals.h:25) */
    double target_distance_m;          /* reference default 0.025 (normals.h:23) */
    double vertical_subtent_rad;       /* > 0: use this instead of deriving it from the first return */
    double* vertical_subtent_out;      /* optional, n_frames doubles: the first return's vertical pixel subtent */
} ob_normals_io;
ob_status ob_normals(ob_dtype dtype, const ob_normals_io* io, ob_stream* s);

/* ---- ground segmentation (DESIGN f-13) ----
 * replaces impl::get_ground_mask / get_ground_mask_into     ouster_algorithm/src/ground_seg.cpp:1137-1314
 *          build_lower_envelope_ground_model and its passes ground_seg.cpp:179-945
 *          GroundSegEngine::update (one call per FrameSet)   ground_seg.cpp:1319-1343
 * One call segments every frame of a set (lut == NULL marks an empty slot, as in ob_dewarp_frames_io); each frame
 * has its own shape, LUT and grid, and grid_size is one value for the call.  The model is built from the first two
 * returns; every return gets a mask (1 = ground), and returns 3 and later are classified without normals.
 * Arithmetic and orders are those of the oracle (oracle/orc_ground.c, DESIGN §9): given the same normals, the
 * model after every pass and every mask pixel are bit-identical to it.
 * normals / normals2: the frame's NORMALS / NORMALS2 fields (float32, h*w x 3, widened exactly); normals2 is read
 * only alongside normals, and a second return without it is classified without normals.  A frame without normals
 * and with compute_normals set gets the normals get_ground_mask computes (ground_seg.cpp:1195-1250): ob_normals with
 * the reference's defaults on the dewarped float64 points of the first two returns, with per-column sensor origins
 * (pose_c * sensor_to_body).translation; those launches count as "normals" (one ob_normals batch per distinct
 * frame shape and return count in the call).  vertical_subtent_out receives the vertical pixel subtent they used
 * (one device acos: the only way such a run can differ from a CPU one, DESIGN §9).  A frame without normals and
 * without compute_normals is segmented without normals.
 * stop: the pass to stop after (OB_GROUND_CELLS .. OB_GROUND_FINAL); the masks are classified only at
 * OB_GROUND_FINAL and are zeroed otherwise.  Masks are written whole.
 * Optional model outputs: the header, and the five grids (rows x cols, row-major) after pass `stop`; grid_capacity
 * is their length in cells.
 * Errors, checked before anything is launched (OB_INVALID_ARGUMENT, the reference's texts): "GroundSegConfig.grid_size
 * must be > 0", then per frame "frame must contain RANGE field for get_ground_mask", "not enough output masks
 * provided for get_ground_mask_into", "output mask shape does not match frame shape"; then OB_NO_DEVICE without a
 * GPU, "ground segmentation needs a float64 lut" and "lut shape does not match frame shape".  The grid shapes are known only on the device: the call waits
 * once for them, then fails "output capacity too small" when a frame's grid outputs are shorter than its grid.  A
 * failing call writes no output.
 * The wait makes the call impossible to capture in a CUDA graph.  Launches (family "ground", not counting CUB's
 * sort and scan kernels): a fixed number for each `stop`, whatever the number of frames (22 at OB_GROUND_FINAL, one
 * more when some frame computes its normals).
 * An item with h * w == 0 has no pixel and is skipped.  Buffers may be host or device memory. */
typedef enum ob_ground_stage {
    OB_GROUND_CELLS = 0,
    OB_GROUND_FILL1 = 1,
    OB_GROUND_SMOOTH1 = 2,
    OB_GROUND_PRUNE = 3,
    OB_GROUND_FILL2 = 4,
    OB_GROUND_SMOOTH2 = 5,
    OB_GROUND_COMPONENTS = 6,
    OB_GROUND_FILL3 = 7,
    OB_GROUND_FINAL = 7
} ob_ground_stage;
typedef struct ob_ground_model {
    double origin_x, origin_y; /* world xy of cell (0, 0)'s corner */
    double fallback_z;         /* NaN without model points */
    double footprint_bound;    /* 95th percentile of max(|x|, |y|); <= 25 m: indoor */
    int32_t rows, cols;        /* 0 x 0 without model points */
    int32_t valid;             /* some cell holds a height */
    int32_t has_columns;       /* some column has status bit 0 */
} ob_ground_model;
typedef struct ob_ground_item {
    const ob_lut* lut;             /* OB_F64, h x w, built with extrinsics; NULL: empty slot */
    size_t h, w;
    const uint32_t* const* range;  /* n_returns range images h x w (RANGE, RANGE2, ...); the array is host memory */
    size_t n_returns;
    const uint32_t* status;        /* w */
    const double* poses;           /* w x 16: body_to_world per column */
    const float* normals;          /* optional h*w x 3 */
    const float* normals2;         /* optional h*w x 3, used only with normals */
    const double* sensor_to_body;  /* 16, row-major: SensorInfo::extrinsic; read only when normals are computed */
    int32_t compute_normals;       /* 1: compute normals when `normals` is NULL (what get_ground_mask does) */
    int32_t pad;
    double* vertical_subtent_out;  /* optional, 1 double: the subtent of the computed normals */
    uint8_t* const* masks;         /* n_masks masks of mask_h x mask_w (the array is host memory) */
    size_t n_masks, mask_h, mask_w;
    ob_ground_model* model;        /* optional */
    uint8_t* valid;                /* optional grids after pass `stop`, rows x cols */
    uint8_t* obstacle;
    double* floor_z;
    double* height;
    double* roughness;
    size_t grid_capacity;          /* cells of each grid output */
    int32_t* prune_levels;         /* optional: BFS levels the prune pass ran (0 when it did not run) */
} ob_ground_item;
ob_status ob_ground_mask(const ob_ground_item* items, size_t n_items, double grid_size, int stop, ob_stream* s);

/* ---- voxel-grid downsampling (SURVEY 8f-2, the prefilter beside normals) ----
 * replaces core::voxel_downsample(frame, voxel_size)      ouster_core/src/voxel_hash_map.cpp:262-310   (SHUFFLE_FIRST)
 *          core::voxel_downsample_3d / _xd(frame, ...)     ouster_core/src/voxel_hash_map.cpp:312-393   (FIRST_N_POINT,
 *                                                          AVERAGE_POINT, RANDOM; voxel_hash_map.h:287-334, 587-635)
 *          algorithm::voxel_downsample_with_normals        ouster_algorithm/src/voxel_downsample.cpp:21-57 (POINT_NORMAL;
 *                                                          PointNormalBucket, voxel_hash_map.h:142-185)
 * Voxel of a row: floor(p * (1.0 / voxel_size)) on columns 0-2, cast to int32 with NaN / out-of-range -> INT32_MIN
 * (x86 cvttsd2si, what the reference compiles to).  float32 inputs are widened exactly; outputs are float64.
 * Output order: SHUFFLE_FIRST is the reference's order exactly (points_out / indices_out); the other modes emit
 * voxels in the order of their first row in the input (the reference: tsl::robin_map iteration order), inside a
 * voxel in the bucket's slot order.  indices_out (optional) = source row of every output row (for AVERAGE_POINT
 * and POINT_NORMAL: the voxel's first row).  Every mode except POINT_NORMAL returns an empty result for an empty
 * input before any check; POINT_NORMAL skips rows with a non-finite point or normal or a normal of norm <= 1e-12.
 * Row count: n (host) or, when n_device is set, a device word read in stream order (values above `capacity` are
 * clamped; work is launched for `capacity` rows, parameters are checked whenever capacity > 0).  n_out may be
 * host memory (the call waits for the count, then for the rows of host outputs, which are final on return) or
 * device memory (nothing waits; all outputs must then be device memory).  Output buffers hold `capacity` (or n)
 * rows.
 * errors (OB_INVALID_ARGUMENT, the reference's std::invalid_argument texts): "max_points_per_voxel must be greater
 * than 0" (checked first), "voxel_size must be greater than 0", "voxel_downsample_xd: frame must have at least 3
 * columns", "voxel_downsample_with_normals expects Nx3 inputs", "voxel_downsample_with_normals voxel_size must be > 0".
 */
typedef enum ob_voxel_mode {
    OB_VOXEL_FIRST_N_POINT = 0, /* VoxelDownsampleStrategy::FIRST_N_POINT */
    OB_VOXEL_AVERAGE_POINT = 1, /* VoxelDownsampleStrategy::AVERAGE_POINT */
    OB_VOXEL_RANDOM = 2,        /* VoxelDownsampleStrategy::RANDOM */
    OB_VOXEL_SHUFFLE_FIRST = 3, /* core::voxel_downsample */
    OB_VOXEL_POINT_NORMAL = 4   /* algorithm::voxel_downsample_with_normals */
} ob_voxel_mode;

typedef struct ob_voxel_io {
    int32_t mode;                /* ob_voxel_mode */
    int32_t dtype;               /* ob_dtype of points / normals */
    const void* points;          /* rows x cols */
    size_t cols;                 /* >= 3 (3 for SHUFFLE_FIRST and POINT_NORMAL); columns 0-2 are x, y, z */
    const void* normals;         /* POINT_NORMAL: rows x 3 */
    size_t n;                    /* row count when n_device is NULL */
    const size_t* n_device;      /* optional device-resident row count (e.g. ob_dewarp_frames' n_points) */
    size_t capacity;             /* rows the input buffers hold; used with n_device */
    double voxel_size;
    size_t max_points_per_voxel; /* FIRST_N_POINT, RANDOM (reference default 1) */
    size_t min_pts_threshold;    /* AVERAGE_POINT (reference default 1) */
    double* points_out;          /* rows x cols float64 (POINT_NORMAL: x 3) */
    double* normals_out;         /* POINT_NORMAL, optional: rows x 3 float64 unit normals */
    uint32_t* indices_out;       /* optional: rows */
    size_t* n_out;               /* rows written; host or device memory */
} ob_voxel_io;
ob_status ob_voxel_downsample(const ob_voxel_io* io, ob_stream* s);

/* ---- frame-to-map registration: device-resident VoxelHashMap3d and ICP (DESIGN f-6) ----
 * Rows of x, y, z: `dtype` (OB_F32 / OB_F64) rows x 3, n rows, or a device-resident row count (n_device, clamped to
 * `capacity`, e.g. the n_out of ob_voxel_downsample).  Outputs are float64.  Buffers may be host or device memory. */
typedef struct ob_point_rows {
    int32_t dtype;
    const void* points;     /* rows x 3 */
    size_t n;               /* row count when n_device is NULL */
    const size_t* n_device; /* optional device-resident row count */
    size_t capacity;        /* rows the buffer holds; used with n_device */
} ob_point_rows;

typedef struct ob_voxel_map ob_voxel_map; /* VoxelHashMap3d / Xd: open-addressing table in device memory */

/* replaces VoxelHashMap3d(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold)
 *          ouster_core/src/voxel_hash_map.cpp:14-41 (min_pts_threshold is stored and unused, as there)
 * errors (OB_INVALID_ARGUMENT, checked in this order): "max_points_per_voxel must be greater than 0",
 * "voxel_size must be greater than 0", "max_distance must be greater than 0"; then OB_NO_DEVICE without a GPU. */
ob_status ob_voxel_map_create(double voxel_size, double max_distance, size_t max_points_per_voxel,
                              size_t min_pts_threshold, int device, ob_voxel_map** out);
/* replaces VoxelHashMapXd(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold, num_attributes)
 *          voxel_hash_map.h:352-517 with Eigen::VectorXd points (DESIGN f-11): every point is 3 + num_attributes
 * doubles, x, y, z first.  Voxels, the first_n_point gate, the cull and every search use x, y, z only; the attributes
 * ride along.  ob_voxel_map_create is this call with num_attributes = 0.  Same errors in the same order, then
 * "num_attributes too large" above 65535. */
ob_status ob_voxel_map_create_xd(double voxel_size, double max_distance, size_t max_points_per_voxel,
                                 size_t min_pts_threshold, size_t num_attributes, int device, ob_voxel_map** out);
/* VoxelHashMap::point_cols(): 3 + num_attributes, the row width of every rows x cols buffer of this map */
ob_status ob_voxel_map_cols(const ob_voxel_map* m, size_t* cols);
ob_status ob_voxel_map_destroy(ob_voxel_map* m);
/* replaces VoxelHashMap::clear                      voxel_hash_map.h:387-389 */
ob_status ob_voxel_map_clear(ob_voxel_map* m, ob_stream* s);
/* replaces VoxelHashMap::add_points / add_point     voxel_hash_map.cpp:85-107, first_n_point voxel_hash_map.h:287-301
 * The result equals inserting the rows one at a time.  Asynchronous unless a host-side bound (occupied slots plus
 * the batch's row capacity, or `capacity` with n_device) passes half the table: then the call synchronises once to
 * read the counters and the batch's distinct-voxel count, and grows the table to the next power of two >=
 * 4 x (live + new voxels) slots (DESIGN 4, f-6).  Growth frees the old table, so a CUDA graph that captured
 * ob_icp_align or ob_voxel_map_closest_neighbors on this map must be captured again.  error (OB_RUNTIME_ERROR):
 * "voxel map: a table of N slots (B bytes) does not fit in free device memory"; on any error the map is unchanged
 * and nothing of the batch is inserted.  A map with attributes refuses this call (OB_INVALID_ARGUMENT,
 * "VoxelHashMap::add_points received unexpected point dimension"): use ob_voxel_map_add_rows. */
ob_status ob_voxel_map_add_points(ob_voxel_map* m, const ob_point_rows* rows, ob_stream* s);

/* float64 rows x cols, n rows or a device-resident row count clamped to `capacity` (e.g. the n_rows of
 * ob_frames_to_map_rows).  Host or device memory. */
typedef struct ob_map_rows {
    const double* rows;     /* rows x cols */
    size_t cols;
    size_t n;               /* row count when n_device is NULL */
    const size_t* n_device; /* optional device-resident row count */
    size_t capacity;        /* rows the buffer holds; used with n_device */
} ob_map_rows;
/* replaces VoxelHashMap::add_points(Eigen::Ref<const ArrayXXdR>)   voxel_hash_map.h:399-411
 * As ob_voxel_map_add_points for rows of any map: the gate reads columns 0-2, an admitted row keeps all its columns,
 * a rejected row's attributes are dropped.  error: cols != 3 + num_attributes gives "VoxelHashMap::add_points
 * received unexpected point dimension" (OB_INVALID_ARGUMENT). */
ob_status ob_voxel_map_add_rows(ob_voxel_map* m, const ob_map_rows* rows, ob_stream* s);

/* replaces remove_voxels_far_from_location / extract_voxels_far_from_location   voxel_hash_map.cpp:109-154
 * origin: 3 doubles, host or device (so a device-resident pose can feed it).  Voxels with
 * |v - v_origin|^2 >= (ceil(max_distance / voxel_size) + 1)^2, in wrapping int32 arithmetic as the reference runs on
 * x86, are erased.  n_extracted != NULL also emits their points (creation order, then slot order) into `extracted`
 * (capacity rows x cols float64, cols = ob_voxel_map_cols; give it at least the map's point count, ob_voxel_map_size):
 * with a host n_extracted the call waits for the count and, for a host `extracted`, then for the rows; more rows
 * than `capacity` fail "output capacity too small" (the voxels are erased regardless) with *n_extracted left 0 and
 * `extracted` untouched.  With a device n_extracted nothing waits, rows past `capacity` are cut and the count is the
 * true total; a host `extracted` is then refused before the cull, leaving the map unchanged.  extracted == NULL
 * counts only. */
typedef struct ob_voxel_map_cull_io {
    const double* origin;
    double* extracted;
    size_t capacity;
    size_t* n_extracted;
} ob_voxel_map_cull_io;
ob_status ob_voxel_map_remove_far(ob_voxel_map* m, const ob_voxel_map_cull_io* io, ob_stream* s);

/* replaces VoxelHashMap::pointcloud / pointcloud_vector   voxel_hash_map.cpp:43-76
 * Voxels in creation order (the reference: tsl::robin_map order, DESIGN 9), inside a voxel in slot order.
 * points: capacity rows x cols float64 (cols = ob_voxel_map_cols; NULL: count only); n_out host or device, with
 * the capacity rule of ob_voxel_map_remove_far's extraction (a count-only call never exceeds it). */
ob_status ob_voxel_map_point_cloud(const ob_voxel_map* m, double* points, size_t capacity, size_t* n_out,
                                   ob_stream* s);
/* live voxels and stored points (VoxelHashMap::empty is voxels == 0); synchronises the stream */
ob_status ob_voxel_map_size(const ob_voxel_map* m, size_t* voxels, size_t* points, ob_stream* s);

/* replaces VoxelHashMap::get_closest_neighbor(query, max_distance_sq), one query per row   voxel_hash_map.cpp:194-247
 * The 27 voxels in VOXEL_SHIFTS order, each pruned by its AABB lower bound, the first strictly smaller squared
 * distance kept; cols zeros and max_distance_sq when nothing qualifies.  Queries are x, y, z.  neighbors: rows x cols
 * float64 (cols = ob_voxel_map_cols: the neighbour's whole point, attributes included); distances_sq (optional): rows
 * float64. */
typedef struct ob_voxel_query_io {
    ob_point_rows queries;
    double max_distance_sq; /* the reference's default is DBL_MAX */
    double* neighbors;
    double* distances_sq;
} ob_voxel_query_io;
ob_status ob_voxel_map_closest_neighbors(const ob_voxel_map* m, const ob_voxel_query_io* io, ob_stream* s);

/* replaces ICPRegistration::align_points_to_map(frame, VoxelHashMap3d / VoxelHashMapXd, max_distance, kernel_scale)
 *          ouster_mapping/src/icp_registration.cpp (align_points_to_map_impl, data_association, build_linear_system)
 * Every iteration runs on the stream: association fused with applying the previous increment to the source,
 * order-preserving compaction, the linear system in parallel_deterministic_reduce's tree, and one kernel for the
 * LDLT solve, SE3::exp, t_icp = estimation * t_icp and the stop test (|dx|^2 < convergence_criterion^2).
 * pose: 16 doubles, row-major 4x4 (t_icp.matrix()); iterations (optional): iterations run, 0 for an empty map
 * (which gives the identity).  Device pose and iterations: nothing waits for the GPU; otherwise one synchronisation. */
typedef struct ob_icp_io {
    ob_point_rows source;
    double max_distance;          /* max correspondence distance */
    double kernel_scale;          /* Geman-McClure scale */
    int32_t max_num_iterations;   /* ICPRegistration::max_num_iterations_ (reference default 50) */
    double convergence_criterion; /* ICPRegistration::convergence_criterion_ (reference default 1e-4) */
    double* pose;
    int32_t* iterations;
} ob_icp_io;
ob_status ob_icp_align(const ob_voxel_map* m, const ob_icp_io* io, ob_stream* s);

/* ---- frame -> map rows: the map exporter's per-return step on the device (DESIGN f-11) ----
 * replaces, for every item (one return of one frame), python/src/ouster/cli/plugins/map_export.py:589-617:
 *   valid = range > 0; dewarp(xyzlut_double(range), body_to_world)[valid], then every field's pixels [valid] as
 *   columns, np.concatenate(..., axis=1).astype(float64)
 * Output rows are [x, y, z | the fields' channels widened to double, in table order], one per pixel with range > 0,
 * in row-major pixel order of the staggered image, item i's rows after item i-1's.  The XYZ is K1's projection and
 * pose arithmetic (bit for bit the ob_cloud_io poses result).  ONE kernel launch (decoupled look-back compaction,
 * as ob_dewarp_frames).  n_rows in host memory: the call waits for the count, then for host rows; "output capacity
 * too small" when more rows than `capacity` pass (n_rows left 0, rows untouched).  n_rows in DEVICE memory (rows in
 * device memory too): nothing waits, and a count above `capacity` means the list was cut there.  Fields are not tone-mapped (the exporter's float16 RGB step).
 * errors: "map rows need a float64 lut", "unknown field type", "field channels must be at least 1",
 * "cols must be 3 plus the channels of every item's fields", "too many fields" (more than 16 per item). */
typedef struct ob_map_field {
    const void* data;  /* h x w x channels pixels, staggered like the range */
    int32_t type;      /* ChanFieldType tag (chanfield.h): 1..10, or 12 for float16 */
    uint32_t channels; /* >= 1 */
} ob_map_field;
typedef struct ob_map_rows_item {
    const ob_lut* lut;          /* float64 (xyzlut_double) */
    const uint32_t* range;      /* h x w, staggered */
    const double* poses;        /* w x 16: body_to_world (row-major 4x4 per column) */
    const ob_map_field* fields; /* host table of n_fields entries */
    size_t n_fields;
} ob_map_rows_item;
ob_status ob_frames_to_map_rows(const ob_map_rows_item* items, size_t n_items, double* rows, size_t cols,
                                size_t capacity, size_t* n_rows, ob_stream* s);

/* replaces build_linear_system(correspondences, kernel_scale)   ouster_mapping/src/icp_registration.cpp
 * source / target: n x 3 float64 pairs (n or a device count clamped to capacity); jtj: 36 doubles row-major (lower
 * triangle filled, the rest 0, as the reference leaves it), jtr: 6 doubles.  Same summation tree as the reference. */
typedef struct ob_icp_system_io {
    const double* source;
    const double* target;
    size_t n;
    const size_t* n_device;
    size_t capacity;
    double kernel_scale;
    double* jtj;
    double* jtr;
} ob_icp_system_io;
ob_status ob_icp_linear_system(const ob_icp_system_io* io, ob_stream* s);

/* ---- cloud-to-cloud ICP (DESIGN f-7) ---- */
typedef enum ob_align_mode { OB_ALIGN_POINT_TO_POINT = 0, OB_ALIGN_POINT_TO_PLANE = 1 } ob_align_mode;

/* replaces algorithm::point_to_point_align and algorithm::point_to_plane_align
 *          ouster_algorithm/src/align_clouds.cpp:1590-1874 (declared in align_clouds.h:20-84), with the
 *          SpatialHashGrid3D they search (align_clouds.cpp:146-235, impl/spatial_hash.h:73-101)
 * source / target: rows of one dtype (a device count works as for ob_icp_align).  POINT_TO_PLANE also reads
 * source_normals / target_normals (rows x 3 of that dtype; *_normal_rows is their row count, which must equal the
 * points' rows: n, or capacity with n_device).  initial_guess: 16 doubles, row-major, host or device (NULL: the
 * identity).  pose: 16 doubles out; iterations (optional): the iterations that reached the solve (the SVD or the
 * LDLT).  At most 10 iterations; fewer than 20 rows in either cloud, or no iteration with 20 correspondences, give
 * initial_guess back bit for bit.  Device pose and iterations: nothing waits for the GPU and the call can be
 * captured in a CUDA graph; otherwise one synchronisation.
 * errors (OB_INVALID_ARGUMENT, checked in this order, before the 20-row rule):
 * "max_corr_dist must be finite and greater than zero", "max_normal_angle_deg must be finite and in [0, 180]",
 * "source_points and source_normals must have the same number of rows",
 * "target_points and target_normals must have the same number of rows"; then OB_NO_DEVICE without a GPU. */
typedef struct ob_cloud_align_io {
    int32_t mode; /* ob_align_mode */
    ob_point_rows source;
    ob_point_rows target;
    const void* source_normals;
    size_t source_normal_rows;
    const void* target_normals;
    size_t target_normal_rows;
    const double* initial_guess;
    double max_corr_dist;        /* reference default 0.25 */
    double max_normal_angle_deg; /* POINT_TO_PLANE; reference default 20 */
    double* pose;
    int32_t* iterations;
} ob_cloud_align_io;
ob_status ob_cloud_align(const ob_cloud_align_io* io, ob_stream* s);

/* replaces SpatialHashGrid3D(target[, target_normals], cell_size).nearest(target, query, max_dist_sq), one query
 *          per row   align_clouds.cpp:170-235
 * Cells are floor(p / cell_size) in int64 (NaN and out-of-range: INT64_MIN, as on x86); target rows that are not
 * finite (or, with target_normals, whose normal is not finite or has norm <= 1e-12) are left out.  The 27 cells in
 * dx, dy, dz order, a cell's rows in ascending index, the first strictly smaller squared distance below
 * max_dist_sq kept.  indices: one int32 per query row, -1 for none (and for a non-finite query).  target and
 * queries share a dtype; target_normals has target's. */
typedef struct ob_cloud_nearest_io {
    ob_point_rows target;
    const void* target_normals; /* optional */
    ob_point_rows queries;
    double cell_size;
    double max_dist_sq;
    int32_t* indices;
} ob_cloud_nearest_io;
ob_status ob_cloud_nearest(const ob_cloud_nearest_io* io, ob_stream* s);

/* ---- global cloud alignment (DESIGN f-14) ---- */
#define OB_ALIGN_COARSE_YAWS 180  /* pass 1: 2 degree steps */
#define OB_ALIGN_FINE_YAWS 7      /* pass 2: 1 degree steps, +-3 degrees around the best coarse yaw */
#define OB_ALIGN_Z_BINS 1024      /* Z histogram: 0.2 m bins */
#define OB_ALIGN_MAX_FINE_BASE 481   /* largest fine grid side (60 m bound, 0.25 m pixels) */
#define OB_ALIGN_MAX_COARSE_BASE 241 /* largest coarse grid side (60 m bound, 0.5 m pixels) */

/* What one ob_align_clouds call decided, for tests and diagnostics.  Z shifts are in 0.2 m bins, dx / dy in fine
 * pixels; scores are the peak of the normalised cross-correlation (0 for an empty grid).  Poses are row-major 4x4.
 * With fewer than 20 feature points in either cloud only the feature counts are set (searched = 0).  The three
 * optional host buffers receive the target's un-normalised BEV grids (row y of the grid is row y of the buffer,
 * base_n x base_n, so they must hold OB_ALIGN_MAX_*_BASE^2 doubles) and its Z histogram. */
typedef struct ob_align_clouds_trace {
    size_t source_features, target_features;
    int32_t searched, coarse_index, fine_index, pad;
    double bound_m, fine_pixel_m, coarse_pixel_m, max_shift_m;
    int32_t fine_base_n, fine_fft_n, fine_max_shift; /* max_shift: the window half-width in pixels */
    int32_t coarse_base_n, coarse_fft_n, coarse_max_shift;
    double coarse_scores[OB_ALIGN_COARSE_YAWS];
    int32_t fine_z_bins[OB_ALIGN_FINE_YAWS], fine_dx[OB_ALIGN_FINE_YAWS], fine_dy[OB_ALIGN_FINE_YAWS], pad2;
    double fine_scores[OB_ALIGN_FINE_YAWS];
    double initial_pose[16]; /* the yaw search's result */
    double icp_poses[48];    /* after the ICP passes at 2.0, 0.6 and 0.25 m */
    double initial_confidence, refined_confidence;
    size_t initial_matched, initial_total, refined_matched, refined_total;
    double stage_ms[5]; /* device time (CUDA events) of features, pass 1 (with the target's grids and the Z shift),
                           pass 2, ICP and confidence */
    double* target_fine_grid;   /* optional */
    double* target_coarse_grid; /* optional */
    double* target_z_hist;      /* optional, OB_ALIGN_Z_BINS doubles */
} ob_align_clouds_trace;

/* replaces the six point-cloud overloads of algorithm::align_clouds
 *          ouster_algorithm/src/align_clouds.cpp:396-1581, 1876-1995, 2601-2651 (declared in align_clouds.h:183-320)
 * source / target: rows of one dtype, host or device, with n or a device-resident count (as ob_cloud_align).
 * *_cols / *_normal_cols: the columns of the caller's arrays (must be 3).  Normals (rows x 3 of the points' dtype)
 * are optional and must be given for both clouds or for neither.  initial_guess: 16 doubles, row-major, host or
 * device (NULL: the identity).  pose: 16 doubles out; confidence (optional): 1 double out, 0 unless
 * compute_confidence.  trace (optional): host ob_align_clouds_trace.
 * The call waits once for the GPU, to read the feature counts, the footprints and the guess that size the grids
 * and the FFT launches, so it cannot be captured in a CUDA graph.  Host outputs (and a trace) are delivered with
 * the usual closing synchronisation.
 * errors (OB_INVALID_ARGUMENT, checked in this order): "source_points must have shape (N, 3)",
 * "source_normals must have shape (N, 3)", "source_points and source_normals must have the same number of rows",
 * the same three for the target, "source_normals and target_normals must both be given or both be omitted";
 * then OB_NO_DEVICE without a GPU. */
typedef struct ob_align_clouds_io {
    ob_point_rows source;
    ob_point_rows target;
    size_t source_cols, target_cols;
    const void* source_normals; /* optional */
    size_t source_normal_rows, source_normal_cols;
    const void* target_normals; /* optional */
    size_t target_normal_rows, target_normal_cols;
    const double* initial_guess;
    int32_t compute_confidence;
    double* pose;
    double* confidence;
    ob_align_clouds_trace* trace;
} ob_align_clouds_io;
ob_status ob_align_clouds(const ob_align_clouds_io* io, ob_stream* s);

/* ---- zone monitoring (DESIGN f-8) ---- */
#define OB_ZONE_MAX_TRIANGLES 2048 /* Zone::MAX_TRIANGLES */
#define OB_ZONE_MAX_LIVE 16        /* zone_common.py MAX_ACTIVE_ZONES */
typedef enum ob_zone_frame { OB_ZONE_FRAME_NONE = 0, OB_ZONE_FRAME_BODY = 1, OB_ZONE_FRAME_SENSOR = 2 } ob_zone_frame;
typedef enum ob_zone_mode { OB_ZONE_MODE_NONE = 0, OB_ZONE_MODE_OCCUPANCY = 1, OB_ZONE_MODE_VACANCY = 2 } ob_zone_mode;

/* one zone of a render: its STL mesh and the Zone fields check_invariants reads */
typedef struct ob_zone_desc {
    const float* triangles; /* host, n_triangles x 9 floats: v0, v1, v2 of each triangle */
    uint32_t n_triangles;
    int32_t coordinate_frame; /* ob_zone_frame */
    uint32_t point_count;
    uint32_t frame_count;
    int32_t mode; /* ob_zone_mode */
} ob_zone_desc;

/* replaces Zone::render(const BeamConfig&) for every zone of a set   ouster_core/src/zone.cpp:63-135, with
 *          Mesh::closest_and_farthest_intersections (mesh.cpp:249-294), Triangle::intersect (triangle.cpp:19-50)
 *          and the bounding sphere (mesh.cpp:41-60).  One launch covers every zone and pixel.
 * body_* / sensor_*: the BeamConfig LUTs (n_rows * n_cols * 3 doubles each, host or device): make_xyz_lut with
 * range unit 0.001 and scale_translation(sensor_to_body) * lidar_to_sensor, or lidar_to_sensor alone
 * (beam_config.cpp:37-45).  body_* may be NULL when the set has no sensor_to_body_transform.
 * near_mm / far_mm: n_zones x n_rows x n_cols uint32 out (host or device).  pixels_with_intersections: n_zones
 * uint32 out (host); a zone with 0 is one Zone::render returns false for.  The call synchronises once.
 * errors, zone by zone in order: the check_invariants texts (OB_INVALID_ARGUMENT) "Zone: point_count must be in
 * [1, 262143]", "Zone: frame_count must be in [1, 65535]", "Zone: mode must be OCCUPANCY or VACANCY",
 * "Zone: STL coordinate frame must be BODY or SENSOR"; the cases Zone::render reports on stderr
 * (OB_INVALID_ARGUMENT) "Zone: Error rendering zone, STL has no triangles.", "Zone: Error rendering zone, STL has
 * too many triangles.", "Zone: Error rendering zone, sensor_to_body_transform not set for BODY coordinate frame.";
 * after the launch (OB_RUNTIME_ERROR) "Zone::render: range overflow" and "Zone: area of rendered zone (N) is
 * smaller than point_count (M) specified in zone." */
typedef struct ob_zone_render_io {
    uint32_t n_rows, n_cols;
    const double* body_direction;
    const double* body_offset;
    const double* sensor_direction;
    const double* sensor_offset;
    const ob_zone_desc* zones;
    uint32_t n_zones;
    uint32_t* near_mm;
    uint32_t* far_mm;
    uint32_t* pixels_with_intersections;
} ob_zone_render_io;
ob_status ob_zone_render(const ob_zone_render_io* io, ob_stream* s);

/* one live zone of a monitor (slot = its index in power_on_live_ids, the bit it sets in the bitmask) */
typedef struct ob_zone_live {
    uint32_t id; /* ZoneState::id */
    int32_t mode; /* ob_zone_mode; ZoneState::trigger_type */
    uint32_t point_count;
    uint32_t frame_count;
    const uint32_t* near_mm; /* n_rows x n_cols, host or device; copied by ob_zone_monitor_create */
    const uint32_t* far_mm;
    uint32_t triggers; /* initial trigger and alert counters (0 for a new monitor) */
    uint32_t alerts;
} ob_zone_live;

#pragma pack(push, 1)
/* ZoneState (ouster_core/include/ouster/core/zone_state.h), 37 bytes */
typedef struct ob_zone_state {
    uint8_t live, id, error_flags, trigger_type, trigger_status;
    uint32_t triggered_frames, count, occlusion_count, invalid_count, max_count;
    uint32_t min_range, max_range, mean_range;
} ob_zone_state;
#pragma pack(pop)

typedef struct ob_zone_monitor ob_zone_monitor;
/* replaces EmulatedZoneMon (python/src/ouster/sdk/core/zone_common.py) with its zone images in device memory.
 * max_count = #(near < far) per zone is counted on the device here.  error: "at most 16 live zones" */
ob_status ob_zone_monitor_create(int device, uint32_t n_rows, uint32_t n_cols, const ob_zone_live* live,
                                 uint32_t n_live, ob_zone_monitor** out);
/* EmulatedZoneMon::calc_triggers(range, bitmask): range n_rows x n_cols uint32 (host or device, e.g. K2's RANGE);
 * bitmask (optional, host or device) gets bit `slot` OR-ed where the zone triggers.  Per zone: count
 * (r > 0 && near <= r <= far), occlusion (r > 0 && r <= near), invalid (r == 0 && near > 0), min / max / exact
 * sum of the triggering ranges; then one thread runs the OCCUPANCY / VACANCY trigger and alert counters and
 * writes the 16 ZoneState records (get_packet()) in device memory.  Device range and bitmask: nothing waits for
 * the GPU and the call can be captured in a CUDA graph. */
ob_status ob_zone_monitor_update(ob_zone_monitor* m, const uint32_t* range, uint32_t* bitmask, ob_stream* s);
/* the 16 ob_zone_state records of the last update (id 255 for slots past n_live) into `out` (16 * 37 bytes, host
 * or device; a host copy synchronises) */
ob_status ob_zone_monitor_states(const ob_zone_monitor* m, void* out, ob_stream* s);
/* per slot (host arrays of n_live, each optional): the trigger and alert counters, and the exact sum of the last
 * update's triggering ranges (EmulatedZoneMon's float64 mean is range_sums / count); synchronises */
ob_status ob_zone_monitor_counters(const ob_zone_monitor* m, uint32_t* triggers, uint32_t* alerts,
                                   uint64_t* range_sums, ob_stream* s);
ob_status ob_zone_monitor_destroy(ob_zone_monitor* m);

/* ---- image post-processing (DESIGN f-9) ----
 * replaces AutoExposure, BeamUniformityCorrector and LocalToneMapper   ouster_core/src/image_processing.cpp
 * One handle holds one processor's state (lo/hi, their damped states, the update counter, the dark count) in
 * device memory; an update reads and writes it only on the stream, so with device buffers nothing waits for the
 * host and a sequence of updates can be captured in a CUDA graph. */
typedef enum ob_image_kind {
    OB_IMAGE_AUTO_EXPOSURE = 0,
    OB_IMAGE_BEAM_UNIFORMITY = 1,
    OB_IMAGE_LOCAL_TONE_MAP = 2
} ob_image_kind;
typedef enum ob_image_layout {
    OB_IMAGE_MONO = 0,   /* rows x cols of dtype, in place (AE, BUC) */
    OB_IMAGE_RGB = 1,    /* rows x cols x 3 of dtype, in place (AE, LTM) */
    OB_IMAGE_RGB_F16 = 2 /* rows x cols x 3 float16 bits in, float32 out, dtype OB_F32 (AE, LTM) */
} ob_image_layout;

/* the constructor arguments; BUC ignores all of them (damping 0.92, update every 8) */
typedef struct ob_image_params {
    double lo_percentile, hi_percentile; /* each in [0, 1) */
    int32_t update_every;                /* >= 1 */
    int32_t color_correct;               /* LTM only */
    double damping;
    double compress_dr_max_lum; /* LTM only; the bool constructor maps true / false to 0.2 / 0.0 */
} ob_image_params;

/* a snapshot of a processor's state (reference member names in brackets) */
typedef struct ob_image_state {
    double lo, hi, lo_state, hi_state; /* [lo_, hi_, lo_state_, hi_state_], -1 until initialised (AE, LTM) */
    int32_t counter;                   /* [counter_] */
    int32_t initialized;               /* [initialized_] (AE, LTM) */
    uint32_t dark_count_rows;          /* [dark_count_.size()] (BUC), 0 before the first update */
    uint32_t reserved;
} ob_image_state;

typedef struct ob_image_proc ob_image_proc;
/* errors: "lo_percentile and hi_percentile must be in [0, 1)", "update_every must be >= 1", "unknown kind" */
ob_status ob_image_proc_create(int device, int kind /* ob_image_kind */, const ob_image_params* params,
                               ob_image_proc** out);
/* one update(image, update_state) of the reference.  MONO / RGB: `out` is the image, updated in place, and `in`
 * is NULL or equal to `out`.  RGB_F16: `in` holds rows x cols x 3 float16 bits, converted into `out` with
 * f16_bits_to_f32_bits_fast_nan_zero before the update.  Host or device buffers; a host image synchronises.
 * errors: "layout not supported by this processor", "image too large", "stream and processor are on different
 * devices" */
ob_status ob_image_proc_update(ob_image_proc* p, int layout /* ob_image_layout */, int dtype /* ob_dtype */,
                               const void* in, void* out, uint32_t rows, uint32_t cols, int update_state,
                               ob_stream* s);
/* synchronising read of the state; dark_count (optional, host) gets min(dark_count_rows, cap) doubles */
ob_status ob_image_proc_state(const ob_image_proc* p, ob_image_state* state, double* dark_count, size_t cap,
                              ob_stream* s);
ob_status ob_image_proc_destroy(ob_image_proc* p);

/* ---- frame operations (DESIGN f-10) ----
 * replaces frame_ops::clip, filter_field, filter_uv, mask   ouster_core/src/frame_ops.cpp:151-286
 *          frame_ops.filter_xyz                             python/src/ouster/sdk/core/frame_ops.py:83-136
 *          frame_ops::select_by_index (pixel rows)          ouster_core/src/frame_ops.cpp:125-138, 296-323
 * ob_frame_mask_fields is one masked write over the pixel fields of a batch of frames of one shape (h x w): every
 * pixel the predicate hits becomes static_cast<T>(invalid) in each target.  The field table lists per frame the
 * targets (first- or second-return predicate), the fields to zero-fill, and the predicate's sources.  Field
 * selection, the reference's error texts and the per-type skip rules are the caller's (the C++ and Python
 * layers); this entry point refuses what it cannot write exactly:
 *  - a NaN / infinite invalid for an integer target, or one the type cannot hold after truncation toward zero
 *    ("invalid value cannot be represented in the field's type"; the reference's cast is undefined there);
 *  - a VALUE source of a type outside u8..f64 ("filter_field requires a pixel field with shape (h, w) to build a
 *    mask").
 * Every argument is checked before anything is launched, so a failing call modifies nothing.
 * Field data, sources and poses may be device, pinned or pageable memory (host buffers are staged and the call
 * synchronises); the shift and row tables are read on the host and travel with the launch, so a call on device
 * buffers never waits for the host and can be captured in a CUDA graph. */
typedef enum ob_frame_predicate {
    OB_FRAME_CLIP = 0,      /* each target's own value: hit unless lower <= (double)v <= upper (NaN: hit) */
    OB_FRAME_VALUE = 1,     /* source value: hit if lower <= (double)v <= upper (filter_field; mask: u8, [0, 0]) */
    OB_FRAME_ROWS = 2,      /* hit if lower <= row < upper (filter_uv "u") */
    OB_FRAME_COLS = 3,      /* hit if lower <= (col + shift[row]) mod w < upper (filter_uv "v") */
    OB_FRAME_XYZ_RANGE = 4, /* hit if lower <= p[axis] <= upper, p = lut(range) (then the column's pose), in the
                             * LUT dtype with the bounds rounded to it (filter_xyz) */
    OB_FRAME_XYZ_POINTS = 5 /* as XYZ_RANGE on given h x w x 3 points of type 9 (f32) or 10 (f64) */
} ob_frame_predicate;
typedef enum ob_frame_role {
    OB_FRAME_TARGET = 0,  /* written where the first-return predicate hits (CLIP: its own predicate) */
    OB_FRAME_TARGET2 = 1, /* written where the second-return predicate hits */
    OB_FRAME_ZERO = 2,    /* every byte set to 0 (elem_bytes: bytes of one pixel, 1 to 65535) */
    OB_FRAME_SOURCE = 3,  /* first-return source: VALUE field, XYZ_RANGE range (u32), XYZ_POINTS points */
    OB_FRAME_SOURCE2 = 4  /* second-return source */
} ob_frame_role;

typedef struct ob_frame_field {
    void* data;          /* h x w pixels (ZERO: h x w x elements; XYZ_POINTS source: h x w x 3) */
    int32_t type;        /* ChanFieldType tag (chanfield.h): 1..10 for targets and VALUE sources */
    int32_t role;        /* ob_frame_role */
    uint32_t frame;      /* frame of the batch this entry belongs to */
    uint32_t elem_bytes; /* ZERO only: bytes of one pixel, extra dims included */
} ob_frame_field;

typedef struct ob_frame_ops_io {
    uint32_t n_frames, h, w;
    int32_t predicate; /* ob_frame_predicate */
    const ob_frame_field* fields; /* host table, any order, at most 512 entries per frame */
    size_t n_fields;
    double lower, upper, invalid;
    const int32_t* pixel_shift_by_row; /* COLS: h entries, host memory */
    const ob_lut* lut;                 /* XYZ_RANGE */
    const void* poses;                 /* XYZ_RANGE, optional: n_frames x w x 16 of the LUT dtype */
    int32_t axis;                      /* XYZ_*: 0, 1 or 2 */
    int32_t reserved;
} ob_frame_ops_io;

/* errors: "unknown frame predicate", "unknown field role", "axis_idx must be in the range [0, 2]",
 * "Frame dimensions do not match lut.", "range must be uint32", "points must be float32 or float64",
 * "target field type is not a numeric pixel type" and the two above.  Launch family "frame_ops". */
ob_status ob_frame_mask_fields(const ob_frame_ops_io* io, ob_stream* s);

/* one selected-rows copy per entry: dst row k = src row rows[k], row_bytes each (extra dims included) */
typedef struct ob_frame_rows_entry {
    const void* src;
    void* dst;
    size_t row_bytes;
    size_t src_rows;
} ob_frame_rows_entry;

typedef struct ob_frame_rows_io {
    const ob_frame_rows_entry* entries; /* host table */
    uint32_t n_entries;
    uint32_t n_rows;       /* at most 2048 */
    const uint32_t* rows;  /* host memory; each < src_rows of every entry */
} ob_frame_rows_io;

/* errors: "row index out of range", "too many rows for one call".  Launch family "frame_ops". */
ob_status ob_frame_select_rows(const ob_frame_rows_io* io, ob_stream* s);

/* ---- fused range -> (XYZ, destaggered range, destaggered XYZ), batched over frames ----
 * One launch performs, for every frame f and return r of the batch, what the reference does as
 * separate passes: lut(range) (xyzlut.h:139-150) and destagger<uint32_t>(range, shifts)
 * (impl/lidar_frame_impl.h:825-834), optionally destagger<T,3>(xyz) (:849-860) and
 * dewarp<T>(xyz, poses) (pose_util.h:37-59).
 * Layout: element (f, r, ...) of an array lives at base + f*frame_stride + r*return_stride
 * (strides in ELEMENTS of that array's scalar type).  NULL outputs are skipped.  Only the pixels are
 * written: bytes between frames and returns (padded strides) are left untouched, in host and in device memory.
 */
typedef struct ob_cloud_io {
    uint32_t n_frames;
    uint32_t n_returns; /* 1 or 2 (RANGE, RANGE2) */
    const uint32_t* range;
    size_t range_frame_stride, range_return_stride;
    void* xyz; /* staggered order, as cartesian() defines: point i = row*w + col */
    size_t xyz_frame_stride, xyz_return_stride;
    uint32_t* range_destaggered;
    size_t rd_frame_stride, rd_return_stride;
    void* xyz_destaggered;
    size_t xd_frame_stride, xd_return_stride;
    /* optional per-column poses, n_frames x w x 16 scalars of the LUT dtype (row-major 4x4 per
     * column, the layout of LidarFrame::body_to_world cast to T): when set, every XYZ output is
     * dewarp<T>(lut(range), poses) (pose_util.h:37-59) -- point (row, col) becomes R_col*p + t_col,
     * zero-range points included (they land on t_col) -- at no extra pass over memory.
     * poses_frame_stride in scalars; 0 = the same w x 16 block for every frame. */
    const void* poses;
    size_t poses_frame_stride;
} ob_cloud_io;

ob_status ob_scan_to_cloud(const ob_lut* lut, const int32_t* pixel_shift_by_row /* h, host */,
                           size_t n_shifts, const ob_cloud_io* io, ob_stream* s);

/* ---- packet field decode (PacketFormat / FrameBatcher pixel work) ----
 * replaces PacketFormat::block_field<T,BlockDim> / col_field<T>  ouster_core/src/parsing.cpp:628-675
 *          FieldDecodeInfo::get<T>                ouster_core/include/ouster/core/field_decode_info.h:41-54
 *          FrameBatcher::parse_by_block / parse_by_col + zero_fields  ouster_core/src/lidar_frame.cpp:1371-1528
 * The host keeps the FrameBatcher state machine (lidar_frame.cpp:1698-1959) and hands the GPU a
 * frame's packets plus a column map; the GPU writes every pixel field of the frame in one pass.
 */
typedef struct ob_field_desc {
    uint32_t offset;    /* FieldDecodeInfo::offset, bytes from the start of a pixel's channel data */
    uint32_t elem_size; /* sizeof(T) of the destination LidarFrame field (1,2,4,8; 6 = 3 x float16) */
    uint64_t mask;      /* FieldDecodeInfo::mask, applied literally (add_custom_profile replaces 0 by the type
                           mask on the host, profile_extension.cpp:147-150) */
    int32_t shift;      /* FieldDecodeInfo::shift (>0 right, <0 left) */
    int32_t range_return; /* r >= 0: this field is the range image of return r (feeds fused XYZ); else -1 */
    uint32_t zero_pattern; /* 16-bit pattern replicated over missing columns: 0, or 0x7e00 for FLOAT16
                              fields (lidar_frame.cpp:1396-1402) */
    uint32_t reserved;
} ob_field_desc;

typedef struct ob_packet_layout {
    uint32_t packet_header_size; /* 32, legacy 0   (parsing.cpp:459) */
    uint32_t col_header_size;    /* 12, legacy 16  (parsing.cpp:460) */
    uint32_t channel_data_size;  /* profile table  (parsing.cpp:327-356) */
    uint32_t col_size;           /* col_header + h*channel_data + col_footer (parsing.cpp:465-466) */
    uint32_t packet_size;        /* lidar_packet_size (parsing.cpp:467-469) */
    uint32_t columns_per_packet;
    uint32_t pixels_per_column;  /* h */
    uint32_t columns_per_frame;  /* w */
    /* column header decode infos (parsing.cpp:499-538): offsets relative to the column start */
    ob_field_desc col_timestamp, col_measurement_id, col_status;
} ob_packet_layout;

ob_status ob_decoder_create(const ob_packet_layout* layout, const ob_field_desc* fields,
                            size_t n_fields, int device, ob_decoder** out);
ob_status ob_decoder_destroy(ob_decoder* dec);

/* One frame worth of work for ob_decode_frames.
 * packets: n_slots buffers of layout.packet_size bytes, packet_stride apart, in ARRIVAL order.
 * col_src[j] (host, w entries) = slot*columns_per_packet + column index of the packet column whose
 *   pixel data lands in frame column j, or -1: column j is zero-filled (missing / invalid / dropped).
 *   NULL means the identity map (slot j/cpp, column j%cpp): a complete in-order frame.
 * The optional device copies of the column headers (timestamp / measurement_id / status) are decoded
 *   from the same packet column as the pixels (col_src).  FrameBatcher writes the LidarFrame's own
 *   header arrays on the host, exactly like the reference, including the corner case where block
 *   parsing meets non-consecutive measurement ids (parsing.cpp:647-653).
 * fields[i]: h x w row-major image of fields[i].elem_size bytes for decoder field i; NULL = skip.
 * Fused consumers (all optional): with lut != NULL, xyz[r] / range_destaggered[r] receive the same
 * products as ob_scan_to_cloud for the range field(s) tagged with range_return = r.
 */
typedef struct ob_decode_io {
    const uint8_t* packets;
    size_t n_slots, packet_stride;
    const int32_t* col_src;
    void* fields[OB_MAX_FIELDS];
    uint64_t* timestamp;      /* w */
    uint16_t* measurement_id; /* w */
    uint32_t* status;         /* w */
    void* xyz[OB_MAX_RETURNS];
    uint32_t* range_destaggered[OB_MAX_RETURNS];
    const ob_lut* lut; /* optional per-frame LUT (frames of different sensors in one launch); must
                          have the dtype of the call-level lut, which it overrides for this frame */
} ob_decode_io;

ob_status ob_decode_frames(const ob_decoder* dec, const ob_decode_io* frames, size_t n_frames,
                           const ob_lut* lut /* nullable */,
                           const int32_t* pixel_shift_by_row /* nullable, h, host */, size_t n_shifts,
                           ob_stream* s);

/* Uniformly strided batch of COMPLETE, in-order frames (identity column map): frame f of every
 * array lives `*_frame_stride` BYTES after frame f-1.  Same products as ob_decode_frames with O(1)
 * host work per call -- the form a packet ring / frame pool uses.
 * Each output is written in its n_frames blocks (one frame's image or header array) and nowhere else, in host
 * and device memory alike: the bytes between two frames' blocks keep their contents, so outputs may interleave
 * in one allocation (K1's [frame][return] XYZ layout, or a pool that holds all outputs of a frame back to back).
 * A host output with such gaps is decoded into dense device scratch and copied back one block per frame. */
typedef struct ob_decode_batch {
    uint32_t n_frames;
    const uint8_t* packets; /* frame f, slot k at packets + f*packets_frame_stride + k*packet_stride */
    size_t n_slots, packet_stride, packets_frame_stride;
    void* fields[OB_MAX_FIELDS];
    size_t field_frame_stride[OB_MAX_FIELDS];
    uint64_t* timestamp;
    uint16_t* measurement_id;
    uint32_t* status;
    size_t timestamp_frame_stride, measurement_id_frame_stride, status_frame_stride;
    void* xyz[OB_MAX_RETURNS];
    size_t xyz_frame_stride;
    uint32_t* range_destaggered[OB_MAX_RETURNS];
    size_t rd_frame_stride;
    const ob_lut* const* frame_luts; /* optional: n_frames LUT handles, one per frame (independent
                                        sensor streams batched into one launch); NULL = call-level lut */
} ob_decode_batch;

ob_status ob_decode_batch_run(const ob_decoder* dec, const ob_decode_batch* batch, const ob_lut* lut,
                              const int32_t* pixel_shift_by_row, size_t n_shifts, ob_stream* s);

/* ---------------------------------------------------------------------------------------------
 * Decode job: ob_decode_frames for ONE frame with persistent device buffers and asynchronous
 * completion, so that a caller (FrameBatcher) can overlap the host state machine of frame k+1 with
 * the H2D / kernel / D2H of frame k.  Replaces the same reference code as ob_decode_frames
 * (lidar_frame.cpp:1422-1528 + finalize :1905-1922); what is new is only the pipelining.
 *
 *   upload(): enqueue the H2D (or D2D) of `count` packets, `src_stride` bytes apart, into packet
 *             slots [first_slot, first_slot+count) of the job.  Page-locked sources are read by
 *             DMA directly -- no bounce copy; uploads_done() blocks until every enqueued upload has
 *             left the source memory.  An upload at first_slot 0 begins a new frame.
 *   submit(): launch the fused decode over slots [0, io->n_slots) (io->packets and
 *             io->packet_stride are ignored) and enqueue the D2H of every host output in `io`;
 *             device output pointers are written in place.  Outputs are valid after wait().
 *             submit() on a busy job waits for the previous submission first.
 * A job is bound to one stream; jobs on different streams overlap (H2D of one with D2H of another).
 * Not thread-safe; one job = one frame in flight.
 */
typedef struct ob_decode_job ob_decode_job;
ob_status ob_decode_job_create(const ob_decoder* dec, size_t reserve_slots, ob_stream* s,
                               ob_decode_job** out);
ob_status ob_decode_job_upload(ob_decode_job* job, const uint8_t* src, size_t src_stride,
                               size_t first_slot, size_t count);
ob_status ob_decode_job_uploads_done(ob_decode_job* job);
ob_status ob_decode_job_submit(ob_decode_job* job, const ob_decode_io* io, const ob_lut* lut,
                               const int32_t* pixel_shift_by_row, size_t n_shifts);
ob_status ob_decode_job_wait(ob_decode_job* job);
int ob_decode_job_busy(const ob_decode_job* job); /* 1 while a submission has not been waited for */
ob_status ob_decode_job_destroy(ob_decode_job* job);

/* ---- K4: LidarFrame fields -> lidar packets (+ CRC64) on the device, the inverse of ob_decode_frames ----
 * replaces impl::frame_to_packets (lidar packets)   ouster_core/include/ouster/core/impl/lidar_frame_impl.h:435-531
 *          PacketFormat::set_block<T>               ouster_core/src/parsing.cpp:1056-1090
 *          FieldDecodeInfo::set<T>                  ouster_core/include/ouster/core/field_decode_info.h:64-78
 *          PacketFormat::calculate_crc (ECMA-182)   ouster_core/src/parsing.cpp:1183-1234
 * `dec` supplies the packet layout and the field table (the same FieldDecodeInfo serves get and set).
 * Per frame: fields[k] = h x w image of decoder field k (NULL: left zero), per-column timestamp / status
 * (measurement_id = column index, as frame_to_packets writes it; columns without status bit 0 get headers
 * but no pixel data, like set_block), and `packet_headers` = the first packet_header_bytes bytes of every
 * packet as the caller's PacketFormat setters wrote them (frame id, init id, serial number, packet type,
 * alert flags, countdowns; >= packet_header_size, may be the whole packet for LEGACY column headers).
 * with_crc != 0 writes the CRC64 of bytes [0, packet_size - 8) into the last 8 bytes (standard headers,
 * non-LEGACY profiles -- the caller decides, as frame_to_packets does at :512-518).  Every one of the
 * w / columns_per_packet packets is produced; dropping packets "with ts == 0 and no valid column"
 * (:497-500) is the caller's (host-side) choice.  Buffers may be host or device memory; the bytes between
 * packets (packet_stride > packet_size) are not written.  Fields are set in decoder order, each clearing
 * its mask's bits first, so where masks overlap the last field wins, as in set_block.  Every field's mask
 * must lie inside its pixel (offset + bytes up to the mask's top bit <= channel_data_size).
 * errors: "Mismatch between expected number of packets and PacketFormat.columns_per_packet". */
typedef struct ob_encode_io {
    const void* fields[OB_MAX_FIELDS];
    const uint64_t* timestamp;
    const uint32_t* status;
    const uint8_t* packet_headers;
    size_t packet_header_bytes;
    uint8_t* packets; /* out: n_packets x packet_stride */
    size_t packet_stride;
} ob_encode_io;
ob_status ob_encode_frames(const ob_decoder* dec, const ob_encode_io* frames, size_t n_frames, int with_crc,
                           ob_stream* s);

/* 0: pageable host memory (or unknown), 1: page-locked host memory, 2: device / managed memory */
int ob_pointer_kind(const void* p);
/* 1 when the CPU may dereference p: anything but plain (non-managed) device memory */
int ob_pointer_host_readable(const void* p);

#ifdef __cplusplus
}
#endif
#endif /* OUSTER_B200_H */
