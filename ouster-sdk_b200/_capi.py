"""ctypes declarations of the C ABI (include/ouster_b200.h).  Loading this module loads
libouster_b200.so; it raises ImportError when the library has not been built -- there is no
Python/CPU fallback for the compute path."""
import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libouster_b200.so")

OB_MAX_FIELDS = 24
OB_MAX_RETURNS = 2
OB_OK, OB_INVALID_ARGUMENT, OB_RUNTIME_ERROR, OB_CUDA_ERROR, OB_NO_DEVICE = range(5)
OB_F32, OB_F64 = 0, 1

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python ouster-sdk_b200/build.py` "
        "(__graft_entry__.build()); the CUDA path has no fallback implementation")

lib = C.CDLL(LIB_PATH)

vp, sz, i32, u32, u64 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint64


class CloudIO(C.Structure):
    _fields_ = [("n_frames", u32), ("n_returns", u32),
                ("range", vp), ("range_frame_stride", sz), ("range_return_stride", sz),
                ("xyz", vp), ("xyz_frame_stride", sz), ("xyz_return_stride", sz),
                ("range_destaggered", vp), ("rd_frame_stride", sz), ("rd_return_stride", sz),
                ("xyz_destaggered", vp), ("xd_frame_stride", sz), ("xd_return_stride", sz),
                ("poses", vp), ("poses_frame_stride", sz)]


class DewarpFrameIO(C.Structure):
    _fields_ = [("range", vp), ("poses", vp), ("status", vp), ("timestamps", vp),
                ("min_range", C.c_double), ("max_range", C.c_double),
                ("points", vp), ("col_idx", vp), ("timestamps_out", vp), ("capacity", sz)]


class NormalsIO(C.Structure):
    _fields_ = [("n_frames", sz), ("h", sz), ("w", sz), ("xyz", vp), ("range", vp), ("xyz2", vp), ("range2", vp),
                ("normals", vp), ("normals2", vp), ("xyz_frame_stride", sz), ("range_frame_stride", sz),
                ("normals_frame_stride", sz), ("sensor_origins_xyz", vp), ("n_origins", sz),
                ("origins_frame_stride", sz), ("pixel_search_range", sz),
                ("min_angle_of_incidence_rad", C.c_double), ("target_distance_m", C.c_double),
                ("vertical_subtent_rad", C.c_double), ("vertical_subtent_out", vp)]


class VoxelIO(C.Structure):
    _fields_ = [("mode", C.c_int32), ("dtype", C.c_int32), ("points", vp), ("cols", sz), ("normals", vp),
                ("n", sz), ("n_device", vp), ("capacity", sz), ("voxel_size", C.c_double),
                ("max_points_per_voxel", sz), ("min_pts_threshold", sz), ("points_out", vp), ("normals_out", vp),
                ("indices_out", vp), ("n_out", vp)]


OB_VOXEL_FIRST_N_POINT, OB_VOXEL_AVERAGE_POINT, OB_VOXEL_RANDOM, OB_VOXEL_SHUFFLE_FIRST, OB_VOXEL_POINT_NORMAL = range(5)


class PointRows(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("points", vp), ("n", sz), ("n_device", vp), ("capacity", sz)]


class MapRows(C.Structure):
    """ob_map_rows"""
    _fields_ = [("rows", vp), ("cols", sz), ("n", sz), ("n_device", vp), ("capacity", sz)]


class MapField(C.Structure):
    """ob_map_field"""
    _fields_ = [("data", vp), ("type", C.c_int32), ("channels", u32)]


class MapRowsItem(C.Structure):
    """ob_map_rows_item"""
    _fields_ = [("lut", vp), ("range", vp), ("poses", vp), ("fields", C.POINTER(MapField)), ("n_fields", sz)]


class InterpPoseIO(C.Structure):
    """ob_interp_pose_io"""
    _fields_ = [("x_interp", vp), ("n", sz), ("x_known", vp), ("m", sz), ("x_dtype", i32), ("pose_dtype", i32),
                ("two_pose", i32), ("pad", i32), ("poses_known", vp), ("poses", vp), ("error", vp)]


class FramePosesItem(C.Structure):
    """ob_frame_poses_item"""
    _fields_ = [("timestamps", vp), ("status", vp), ("poses", vp), ("w", sz)]


OB_POSE_OK, OB_POSE_KNOT_ORDER, OB_POSE_ZERO_DURATION, OB_POSE_DESCENT = range(4)


class GroundModel(C.Structure):
    """ob_ground_model"""
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("fallback_z", C.c_double),
                ("footprint_bound", C.c_double), ("rows", i32), ("cols", i32), ("valid", i32), ("has_columns", i32)]


class GroundItem(C.Structure):
    """ob_ground_item"""
    _fields_ = [("lut", vp), ("h", sz), ("w", sz), ("range", C.POINTER(vp)), ("n_returns", sz), ("status", vp),
                ("poses", vp), ("normals", vp), ("normals2", vp), ("sensor_to_body", vp), ("compute_normals", i32),
                ("pad", i32), ("vertical_subtent_out", vp), ("masks", C.POINTER(vp)), ("n_masks", sz),
                ("mask_h", sz), ("mask_w", sz), ("model", vp), ("valid", vp), ("obstacle", vp), ("floor_z", vp),
                ("height", vp), ("roughness", vp), ("grid_capacity", sz), ("prune_levels", vp)]


# passes of ob_ground_mask's model, in order (ob_ground_stage)
GROUND_STAGES = ("cells", "fill1", "smooth1", "prune", "fill2", "smooth2", "components", "fill3")
OB_GROUND_FINAL = len(GROUND_STAGES) - 1


class VoxelMapCullIO(C.Structure):
    _fields_ = [("origin", vp), ("extracted", vp), ("capacity", sz), ("n_extracted", vp)]


class VoxelQueryIO(C.Structure):
    _fields_ = [("queries", PointRows), ("max_distance_sq", C.c_double), ("neighbors", vp), ("distances_sq", vp)]


class IcpIO(C.Structure):
    _fields_ = [("source", PointRows), ("max_distance", C.c_double), ("kernel_scale", C.c_double),
                ("max_num_iterations", C.c_int32), ("convergence_criterion", C.c_double), ("pose", vp),
                ("iterations", vp)]


class IcpSystemIO(C.Structure):
    _fields_ = [("source", vp), ("target", vp), ("n", sz), ("n_device", vp), ("capacity", sz),
                ("kernel_scale", C.c_double), ("jtj", vp), ("jtr", vp)]


OB_ALIGN_POINT_TO_POINT, OB_ALIGN_POINT_TO_PLANE = range(2)


class CloudAlignIO(C.Structure):
    _fields_ = [("mode", C.c_int32), ("source", PointRows), ("target", PointRows), ("source_normals", vp),
                ("source_normal_rows", sz), ("target_normals", vp), ("target_normal_rows", sz),
                ("initial_guess", vp), ("max_corr_dist", C.c_double), ("max_normal_angle_deg", C.c_double),
                ("pose", vp), ("iterations", vp)]


OB_ALIGN_COARSE_YAWS, OB_ALIGN_FINE_YAWS, OB_ALIGN_Z_BINS = 180, 7, 1024
OB_ALIGN_MAX_FINE_BASE, OB_ALIGN_MAX_COARSE_BASE = 481, 241


class AlignCloudsTrace(C.Structure):
    """ob_align_clouds_trace"""
    _fields_ = [("source_features", sz), ("target_features", sz),
                ("searched", C.c_int32), ("coarse_index", C.c_int32), ("fine_index", C.c_int32), ("pad", C.c_int32),
                ("bound_m", C.c_double), ("fine_pixel_m", C.c_double), ("coarse_pixel_m", C.c_double),
                ("max_shift_m", C.c_double),
                ("fine_base_n", C.c_int32), ("fine_fft_n", C.c_int32), ("fine_max_shift", C.c_int32),
                ("coarse_base_n", C.c_int32), ("coarse_fft_n", C.c_int32), ("coarse_max_shift", C.c_int32),
                ("coarse_scores", C.c_double * OB_ALIGN_COARSE_YAWS),
                ("fine_z_bins", C.c_int32 * OB_ALIGN_FINE_YAWS), ("fine_dx", C.c_int32 * OB_ALIGN_FINE_YAWS),
                ("fine_dy", C.c_int32 * OB_ALIGN_FINE_YAWS), ("pad2", C.c_int32),
                ("fine_scores", C.c_double * OB_ALIGN_FINE_YAWS),
                ("initial_pose", C.c_double * 16), ("icp_poses", C.c_double * 48),
                ("initial_confidence", C.c_double), ("refined_confidence", C.c_double),
                ("initial_matched", sz), ("initial_total", sz), ("refined_matched", sz), ("refined_total", sz),
                ("stage_ms", C.c_double * 5), ("target_fine_grid", vp), ("target_coarse_grid", vp), ("target_z_hist", vp)]


class AlignCloudsIO(C.Structure):
    """ob_align_clouds_io"""
    _fields_ = [("source", PointRows), ("target", PointRows), ("source_cols", sz), ("target_cols", sz),
                ("source_normals", vp), ("source_normal_rows", sz), ("source_normal_cols", sz),
                ("target_normals", vp), ("target_normal_rows", sz), ("target_normal_cols", sz),
                ("initial_guess", vp), ("compute_confidence", C.c_int32), ("pose", vp), ("confidence", vp),
                ("trace", C.POINTER(AlignCloudsTrace))]


class CloudNearestIO(C.Structure):
    _fields_ = [("target", PointRows), ("target_normals", vp), ("queries", PointRows), ("cell_size", C.c_double),
                ("max_dist_sq", C.c_double), ("indices", vp)]


OB_ZONE_MAX_TRIANGLES, OB_ZONE_MAX_LIVE = 2048, 16
OB_ZONE_FRAME_NONE, OB_ZONE_FRAME_BODY, OB_ZONE_FRAME_SENSOR = range(3)
OB_ZONE_MODE_NONE, OB_ZONE_MODE_OCCUPANCY, OB_ZONE_MODE_VACANCY = range(3)


class ZoneDesc(C.Structure):
    _fields_ = [("triangles", vp), ("n_triangles", u32), ("coordinate_frame", C.c_int32), ("point_count", u32),
                ("frame_count", u32), ("mode", C.c_int32)]


class ZoneRenderIO(C.Structure):
    _fields_ = [("n_rows", u32), ("n_cols", u32), ("body_direction", vp), ("body_offset", vp),
                ("sensor_direction", vp), ("sensor_offset", vp), ("zones", C.POINTER(ZoneDesc)), ("n_zones", u32),
                ("near_mm", vp), ("far_mm", vp), ("pixels_with_intersections", vp)]


class ZoneLive(C.Structure):
    _fields_ = [("id", u32), ("mode", C.c_int32), ("point_count", u32), ("frame_count", u32), ("near_mm", vp),
                ("far_mm", vp), ("triggers", u32), ("alerts", u32)]


class ZoneState(C.Structure):
    _pack_ = 1
    _fields_ = [("live", C.c_uint8), ("id", C.c_uint8), ("error_flags", C.c_uint8), ("trigger_type", C.c_uint8),
                ("trigger_status", C.c_uint8), ("triggered_frames", u32), ("count", u32), ("occlusion_count", u32),
                ("invalid_count", u32), ("max_count", u32), ("min_range", u32), ("max_range", u32),
                ("mean_range", u32)]


OB_IMAGE_AUTO_EXPOSURE, OB_IMAGE_BEAM_UNIFORMITY, OB_IMAGE_LOCAL_TONE_MAP = range(3)
OB_IMAGE_MONO, OB_IMAGE_RGB, OB_IMAGE_RGB_F16 = range(3)


class ImageParams(C.Structure):
    _fields_ = [("lo_percentile", C.c_double), ("hi_percentile", C.c_double), ("update_every", C.c_int32),
                ("color_correct", C.c_int32), ("damping", C.c_double), ("compress_dr_max_lum", C.c_double)]


class ImageState(C.Structure):
    _fields_ = [("lo", C.c_double), ("hi", C.c_double), ("lo_state", C.c_double), ("hi_state", C.c_double),
                ("counter", C.c_int32), ("initialized", C.c_int32), ("dark_count_rows", u32), ("reserved", u32)]


OB_FRAME_CLIP, OB_FRAME_VALUE, OB_FRAME_ROWS, OB_FRAME_COLS, OB_FRAME_XYZ_RANGE, OB_FRAME_XYZ_POINTS = range(6)
OB_FRAME_TARGET, OB_FRAME_TARGET2, OB_FRAME_ZERO, OB_FRAME_SOURCE, OB_FRAME_SOURCE2 = range(5)


class FrameField(C.Structure):
    """ob_frame_field"""
    _fields_ = [("data", vp), ("type", C.c_int32), ("role", C.c_int32), ("frame", u32), ("elem_bytes", u32)]


class FrameOpsIO(C.Structure):
    """ob_frame_ops_io"""
    _fields_ = [("n_frames", u32), ("h", u32), ("w", u32), ("predicate", C.c_int32), ("fields", C.POINTER(FrameField)),
                ("n_fields", sz), ("lower", C.c_double), ("upper", C.c_double), ("invalid", C.c_double),
                ("pixel_shift_by_row", C.POINTER(C.c_int32)), ("lut", vp), ("poses", vp), ("axis", C.c_int32),
                ("reserved", C.c_int32)]


class FrameRowsEntry(C.Structure):
    """ob_frame_rows_entry"""
    _fields_ = [("src", vp), ("dst", vp), ("row_bytes", sz), ("src_rows", sz)]


class FrameRowsIO(C.Structure):
    """ob_frame_rows_io"""
    _fields_ = [("entries", C.POINTER(FrameRowsEntry)), ("n_entries", u32), ("n_rows", u32),
                ("rows", C.POINTER(u32))]


class DewarpFramesIO(C.Structure):
    _fields_ = [("lut", vp), ("range", vp), ("poses", vp), ("status", vp), ("timestamps", vp)]


class FieldDesc(C.Structure):
    _fields_ = [("offset", u32), ("elem_size", u32), ("mask", u64), ("shift", C.c_int32),
                ("range_return", C.c_int32), ("zero_pattern", u32), ("reserved", u32)]


class PacketLayout(C.Structure):
    _fields_ = [("packet_header_size", u32), ("col_header_size", u32), ("channel_data_size", u32),
                ("col_size", u32), ("packet_size", u32), ("columns_per_packet", u32),
                ("pixels_per_column", u32), ("columns_per_frame", u32),
                ("col_timestamp", FieldDesc), ("col_measurement_id", FieldDesc),
                ("col_status", FieldDesc)]


class DecodeIO(C.Structure):
    _fields_ = [("packets", vp), ("n_slots", sz), ("packet_stride", sz),
                ("col_src", vp),
                ("fields", vp * OB_MAX_FIELDS),
                ("timestamp", vp), ("measurement_id", vp), ("status", vp),
                ("xyz", vp * OB_MAX_RETURNS), ("range_destaggered", vp * OB_MAX_RETURNS),
                ("lut", vp)]


class DecodeBatch(C.Structure):
    _fields_ = [("n_frames", u32), ("packets", vp), ("n_slots", sz), ("packet_stride", sz),
                ("packets_frame_stride", sz),
                ("fields", vp * OB_MAX_FIELDS), ("field_frame_stride", sz * OB_MAX_FIELDS),
                ("timestamp", vp), ("measurement_id", vp), ("status", vp),
                ("timestamp_frame_stride", sz), ("measurement_id_frame_stride", sz),
                ("status_frame_stride", sz),
                ("xyz", vp * OB_MAX_RETURNS), ("xyz_frame_stride", sz),
                ("range_destaggered", vp * OB_MAX_RETURNS), ("rd_frame_stride", sz),
                ("frame_luts", C.POINTER(vp))]


class EncodeIO(C.Structure):
    _fields_ = [("fields", vp * OB_MAX_FIELDS), ("timestamp", vp), ("status", vp), ("packet_headers", vp),
                ("packet_header_bytes", sz), ("packets", vp), ("packet_stride", sz)]


def _sig(name, restype, *argtypes):
    f = getattr(lib, name)
    f.restype = restype
    f.argtypes = list(argtypes)
    return f


_sig("ob_abi_version", i32)
_sig("ob_abi_sizeof", sz, C.c_char_p)
_sig("ob_last_error", C.c_char_p)
_sig("ob_device_count", i32)
_sig("ob_kernel_launch_count", u64)
_sig("ob_kernel_launch_count_of", u64, C.c_char_p)
_sig("ob_set_tunable", i32, i32, C.c_char_p, i32)
_sig("ob_stream_create", i32, i32, C.POINTER(vp))
_sig("ob_stream_wrap", i32, i32, vp, C.POINTER(vp))
_sig("ob_stream_sync", i32, vp)
_sig("ob_stream_cuda_handle", vp, vp)
_sig("ob_stream_destroy", i32, vp)
_sig("ob_host_alloc", i32, sz, C.POINTER(vp))
_sig("ob_host_free", i32, vp)
_sig("ob_lut_create", i32, i32, vp, vp, sz, sz, i32, C.POINTER(vp))
_sig("ob_lut_from_intrinsics", i32, i32, sz, sz, C.c_double, vp, vp, vp, sz, vp, sz, i32,
     C.POINTER(vp))
_sig("ob_lut_download", i32, vp, vp, vp)
_sig("ob_lut_info", i32, vp, C.POINTER(sz), C.POINTER(sz), C.POINTER(i32), C.POINTER(i32))
_sig("ob_lut_device_ptrs", i32, vp, C.POINTER(vp), C.POINTER(vp))
_sig("ob_lut_destroy", i32, vp)
_sig("ob_lut_set_analytic", i32, vp, i32)
_sig("ob_lut_is_analytic", i32, vp)
_sig("ob_cartesian", i32, vp, vp, sz, vp, vp)
_sig("ob_destagger", i32, sz, sz, vp, vp, sz, sz, sz, i32, vp, vp)
_sig("ob_dewarp", i32, i32, vp, vp, sz, sz, vp, vp)
_sig("ob_scan_to_cloud", i32, vp, vp, sz, C.POINTER(CloudIO), vp)
_sig("ob_dewarp_frame", i32, vp, C.POINTER(DewarpFrameIO), C.POINTER(sz), vp)
_sig("ob_normals", i32, i32, C.POINTER(NormalsIO), vp)
_sig("ob_voxel_downsample", i32, C.POINTER(VoxelIO), vp)
_sig("ob_voxel_map_create", i32, C.c_double, C.c_double, sz, sz, i32, C.POINTER(vp))
_sig("ob_voxel_map_create_xd", i32, C.c_double, C.c_double, sz, sz, sz, i32, C.POINTER(vp))
_sig("ob_voxel_map_cols", i32, vp, C.POINTER(sz))
_sig("ob_voxel_map_add_rows", i32, vp, C.POINTER(MapRows), vp)
_sig("ob_frames_to_map_rows", i32, C.POINTER(MapRowsItem), sz, vp, sz, sz, vp, vp)
_sig("ob_voxel_map_destroy", i32, vp)
_sig("ob_interp_pose", i32, C.POINTER(InterpPoseIO), vp)
_sig("ob_frames_interp_pose", i32, C.POINTER(FramePosesItem), sz, C.c_double, vp, C.c_double, vp, vp, vp)
_sig("ob_ground_mask", i32, C.POINTER(GroundItem), sz, C.c_double, i32, vp)
_sig("ob_voxel_map_clear", i32, vp, vp)
_sig("ob_voxel_map_add_points", i32, vp, C.POINTER(PointRows), vp)
_sig("ob_voxel_map_remove_far", i32, vp, C.POINTER(VoxelMapCullIO), vp)
_sig("ob_voxel_map_point_cloud", i32, vp, vp, sz, vp, vp)
_sig("ob_voxel_map_size", i32, vp, C.POINTER(sz), C.POINTER(sz), vp)
_sig("ob_voxel_map_closest_neighbors", i32, vp, C.POINTER(VoxelQueryIO), vp)
_sig("ob_icp_align", i32, vp, C.POINTER(IcpIO), vp)
_sig("ob_icp_linear_system", i32, C.POINTER(IcpSystemIO), vp)
_sig("ob_cloud_align", i32, C.POINTER(CloudAlignIO), vp)
_sig("ob_cloud_nearest", i32, C.POINTER(CloudNearestIO), vp)
_sig("ob_align_clouds", i32, C.POINTER(AlignCloudsIO), vp)
_sig("ob_zone_render", i32, C.POINTER(ZoneRenderIO), vp)
_sig("ob_zone_monitor_create", i32, i32, u32, u32, C.POINTER(ZoneLive), u32, C.POINTER(vp))
_sig("ob_zone_monitor_update", i32, vp, vp, vp, vp)
_sig("ob_zone_monitor_states", i32, vp, vp, vp)
_sig("ob_zone_monitor_counters", i32, vp, vp, vp, vp, vp)
_sig("ob_zone_monitor_destroy", i32, vp)
_sig("ob_image_proc_create", i32, i32, i32, C.POINTER(ImageParams), C.POINTER(vp))
_sig("ob_image_proc_update", i32, vp, i32, i32, vp, vp, u32, u32, i32, vp)
_sig("ob_image_proc_state", i32, vp, C.POINTER(ImageState), vp, sz, vp)
_sig("ob_image_proc_destroy", i32, vp)
_sig("ob_frame_mask_fields", i32, C.POINTER(FrameOpsIO), vp)
_sig("ob_frame_select_rows", i32, C.POINTER(FrameRowsIO), vp)
_sig("ob_dewarp_frames", i32, C.POINTER(DewarpFramesIO), sz, C.c_double, C.c_double, vp, sz, vp, vp, vp,
     C.POINTER(sz), C.POINTER(sz), vp)
if hasattr(lib, "ob_decoder_create"):
    _sig("ob_decoder_create", i32, C.POINTER(PacketLayout), C.POINTER(FieldDesc), sz, i32,
         C.POINTER(vp))
    _sig("ob_decoder_destroy", i32, vp)
    _sig("ob_decode_frames", i32, vp, C.POINTER(DecodeIO), sz, vp, vp, sz, vp)
    _sig("ob_decode_batch_run", i32, vp, C.POINTER(DecodeBatch), vp, vp, sz, vp)
    _sig("ob_encode_frames", i32, vp, C.POINTER(EncodeIO), sz, i32, vp)


class OusterB200Error(RuntimeError):
    pass


def check(status):
    """Map an ob_status to the exception type the reference raises through its Python binding
    (std::invalid_argument -> ValueError, python/tests/test_xyzlut.py:29-51)."""
    if status == OB_OK:
        return
    msg = lib.ob_last_error().decode()
    if status == OB_INVALID_ARGUMENT:
        raise ValueError(msg)
    raise OusterB200Error(f"[status {status}] {msg}")
