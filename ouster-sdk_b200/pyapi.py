"""Python drop-in for the hot-path part of `ouster.sdk.core` (SURVEY 8f #4): same call shapes and
error behaviour as the nanobind binding (python/src/cpp/client/processing.cpp:340-357, 527-700):

    from ouster_sdk_b200 import pyapi as core
    xyz = core.XYZLut(info)(scan)                 # (H, W, 3) float64, staggered
    img = core.destagger(info, scan.field("RANGE"))
"""
import enum

import numpy as np

from . import core as _c
from .host import FrameBatcher, LidarFrame, LidarScan, ScanBatcher, SensorInfo  # noqa: F401

# ---- device-resident data (SURVEY 8f #4) -----------------------------------------------------------
# Every function below also takes torch CUDA tensors, or any object exporting __dlpack__ from device
# memory, and then returns a torch CUDA tensor (itself a DLPack exporter): a caller can chain
# DeviceScanBatcher -> XYZLut -> destagger -> normals without the data ever leaving HBM.


def _torch():
    import torch
    return torch


def _dev(x):
    """torch CUDA tensor view of `x` when it lives on a GPU (torch tensor or DLPack exporter), else None."""
    if isinstance(x, np.ndarray) or x is None:
        return None
    if _c._is_torch(x):
        return x if x.is_cuda else None
    if hasattr(x, "__dlpack__") and hasattr(x, "__dlpack_device__"):
        kind = int(x.__dlpack_device__()[0])
        if kind in (2, 13):          # kDLCUDA, kDLCUDAManaged
            return _torch().from_dlpack(x)
    return None


class ChanField:
    RANGE, RANGE2, SIGNAL, SIGNAL2 = "RANGE", "RANGE2", "SIGNAL", "SIGNAL2"
    REFLECTIVITY, REFLECTIVITY2, NEAR_IR = "REFLECTIVITY", "REFLECTIVITY2", "NEAR_IR"
    FLAGS, FLAGS2, WINDOW = "FLAGS", "FLAGS2", "WINDOW"
    NORMALS, NORMALS2, GROUND, GROUND2 = "NORMALS", "NORMALS2", "GROUND", "GROUND2"


def _info_dict(info):
    return {"w": info.w, "h": info.h, "beam_to_lidar_transform": info.beam_to_lidar_transform,
            "lidar_to_sensor_transform": info.lidar_to_sensor_transform,
            "sensor_to_body": getattr(info, "sensor_to_body", None),
            "beam_azimuth_angles": info.beam_azimuth_angles,
            "beam_altitude_angles": info.beam_altitude_angles}


class _XYZLutBase:
    _dtype = np.float64

    def __init__(self, info, use_extrinsics=True, device=0):
        self._lut = _c.XYZLutT.from_sensor_info(_info_dict(info), use_extrinsics, self._dtype, device)
        self.h, self.w = self._lut.h, self._lut.w

    @property
    def direction(self):
        return self._lut.direction

    @property
    def offset(self):
        return self._lut.offset

    def __call__(self, scan_or_range):
        """lut(scan) / lut(range image) -> (H, W, 3).  Raises ValueError on a dimension mismatch
        ("Frame dimensions do not match lut." / "Image dimensions do not match lut.")."""
        is_scan = hasattr(scan_or_range, "field")
        rng = scan_or_range.field("RANGE") if is_scan else scan_or_range
        t = _dev(rng)
        if t is not None:   # device range image -> device points
            if tuple(t.shape) != (self.h, self.w):
                raise ValueError("Frame dimensions do not match lut." if is_scan else "Image dimensions do not match lut.")
            torch = _torch()
            if t.dtype not in (torch.int32, torch.uint32):
                raise ValueError("range must be uint32")
            return _c.cartesian(self._lut, t.contiguous().view(torch.uint32)).reshape(self.h, self.w, 3)
        if is_scan:
            if rng.shape != (self.h, self.w):
                raise ValueError("Frame dimensions do not match lut.")
        else:
            rng = np.asarray(scan_or_range)
            if rng.shape != (self.h, self.w):
                raise ValueError("Image dimensions do not match lut.")
        return self._lut(np.ascontiguousarray(rng, np.uint32)).reshape(self.h, self.w, 3)


class XYZLut(_XYZLutBase):
    _dtype = np.float64


class XYZLutFloat(_XYZLutBase):
    _dtype = np.float32


def destagger(info, fields, inverse=False):
    """core.destagger(info, fields, inverse=False): (H, W) or (H, W, k) array of any numeric dtype;
    dtype and shape are preserved; ValueError when the shape does not match the sensor."""
    t = _dev(fields)
    if t is not None:   # device image -> device image (same dtype / shape)
        if t.dim() < 2 or t.dim() > 3:
            raise ValueError("Invalid dimensions for destaggering")
        if t.shape[0] != info.h or t.shape[1] != info.w or t.numel() == 0:
            raise ValueError("Image resolution must match SensorInfo.")
        return _c.destagger(t.contiguous(), info.pixel_shift_by_row, inverse)
    a = np.asarray(fields)
    if a.ndim < 2 or a.ndim > 3:
        raise ValueError("Invalid dimensions for destaggering")
    if a.shape[0] != info.h or a.shape[1] != info.w or a.size == 0:
        raise ValueError("Image resolution must match SensorInfo.")
    if a.dtype == np.bool_:
        return destagger(info, a.view(np.uint8), inverse).view(np.bool_)
    return _c.destagger(np.ascontiguousarray(a), info.pixel_shift_by_row, inverse)


def stagger(info, fields):
    return destagger(info, fields, True)


def _floating(a, what):
    a = np.asarray(a)
    if a.dtype.kind != "f":
        raise TypeError(f"{what} must be floating-point arrays")
    return a


def dewarp(points, poses):
    """core.dewarp(points (H, W, 3), poses (W, 4, 4)) -> (H, W, 3) (processing.cpp:132-161, 300-310):
    float32 points stay float32, anything else is computed in float64; TypeError for non-floating
    input, RuntimeError when W differs."""
    tp = _dev(points)
    if tp is not None:   # device points (+ host or device poses) -> device points
        torch = _torch()
        if not tp.dtype.is_floating_point:
            raise TypeError("points and poses must be floating-point arrays")
        dt = torch.float32 if tp.dtype == torch.float32 else torch.float64
        tq = _dev(poses)
        tq = tq.to(dt) if tq is not None else torch.as_tensor(np.ascontiguousarray(poses), dtype=dt, device=tp.device)
        return _c.dewarp(tp.to(dt).contiguous(), tq.contiguous())
    p, q = _floating(points, "points and poses"), _floating(poses, "points and poses")
    dt = np.float32 if p.dtype == np.float32 else np.float64
    return _c.dewarp(np.ascontiguousarray(p, dt), np.ascontiguousarray(q, dt))


def transform(points, pose):
    """core.transform(points (..., 3), pose (4, 4)) (processing.cpp:312-329)."""
    p, q = _floating(points, "points and pose"), _floating(pose, "points and pose")
    dt = np.float32 if p.dtype == np.float32 else np.float64
    return _c.transform(np.ascontiguousarray(p, dt), np.ascontiguousarray(q, dt))


def normals(xyz, range, *args, **kwargs):
    """algorithm.normals(xyz, range[, xyz2, range2], sensor_origins_xyz, pixel_search_range=1,
    min_angle_of_incidence_rad=1 deg, target_distance_m=0.025) -- python binding of
    ouster_algorithm/include/ouster/algorithm/normals.h:58-108.  Device inputs give device outputs."""
    t = _dev(xyz)
    if t is None:
        return _c.normals(xyz, range, *args, **kwargs)
    torch = _torch()
    conv = [(_dev(a) if _dev(a) is not None else a) for a in args]
    conv = [torch.as_tensor(np.ascontiguousarray(a, np.float64), device=t.device)
            if isinstance(a, np.ndarray) and a.ndim == 2 and a.shape[-1] == 3 else a for a in conv]
    if "sensor_origins_xyz" in kwargs and isinstance(kwargs["sensor_origins_xyz"], np.ndarray):
        kwargs["sensor_origins_xyz"] = torch.as_tensor(np.ascontiguousarray(kwargs["sensor_origins_xyz"], np.float64),
                                                       device=t.device)
    return _c.normals(t.contiguous(), _dev(range), *conv, **kwargs)


class VoxelDownsampleStrategy(enum.IntEnum):
    """core.VoxelDownsampleStrategy (voxel_hash_map.h:697-701, processing.cpp:959-962)."""
    FIRST_N_POINT = 0
    AVERAGE_POINT = 1
    RANDOM = 2


_STRATEGY_MODE = {VoxelDownsampleStrategy.FIRST_N_POINT: "first_n", VoxelDownsampleStrategy.AVERAGE_POINT: "average",
                  VoxelDownsampleStrategy.RANDOM: "random"}


def _voxel_xd(frame, voxel_size, max_points_per_voxel, min_pts_threshold, strategy, name, shape_ok, shape_msg):
    t = _dev(frame)
    f = t.contiguous() if t is not None else np.ascontiguousarray(frame, np.float64)
    if len(f.shape) != 2 or not shape_ok(int(f.shape[1])):
        raise ValueError(shape_msg)
    if f.shape[0] == 0:   # empty frame: returned before any other check (voxel_hash_map.cpp:317, 355)
        return f[:0].double() if t is not None else np.empty((0, f.shape[1]), np.float64)
    try:
        mode = _STRATEGY_MODE[VoxelDownsampleStrategy(strategy)]
    except ValueError:
        raise ValueError(f"{name}: unknown strategy") from None
    return _c.voxel_downsample(f, voxel_size, mode, max_points_per_voxel=max_points_per_voxel,
                               min_pts_threshold=min_pts_threshold)[0]


def voxel_downsample_3d(frame, voxel_size, max_points_per_voxel=1, min_pts_threshold=1,
                        strategy=VoxelDownsampleStrategy.RANDOM):
    """core.voxel_downsample_3d (processing.cpp:511-523, 964-980): Nx3 in, Mx3 float64 out.  Device tensors
    give device tensors.  Voxels come out in first-appearance order (the reference: hash-map order)."""
    return _voxel_xd(frame, voxel_size, max_points_per_voxel, min_pts_threshold, strategy, "voxel_downsample_3d",
                     lambda c: c == 3, "voxel_downsample_3d: frame must be Nx3")


def voxel_downsample_xd(frame, voxel_size, max_points_per_voxel=1, min_pts_threshold=1,
                        strategy=VoxelDownsampleStrategy.RANDOM):
    """core.voxel_downsample_xd (processing.cpp:496-509, 982-990): NxD (D >= 3, columns 0-2 are x, y, z, the
    rest attributes carried along) in, MxD float64 out."""
    return _voxel_xd(frame, voxel_size, max_points_per_voxel, min_pts_threshold, strategy, "voxel_downsample_xd",
                     lambda c: c >= 3, "voxel_downsample_xd: frame must be Nx>=3 (x,y,z + optional attributes)")


voxel_downsample = voxel_downsample_xd   # python/src/ouster/sdk/core/__init__.py:76-78


def voxel_downsample_with_normals(points, normals, voxel_size):
    """algorithm.voxel_downsample_with_normals(points, normals, voxel_size) (voxel_downsample.cpp:21-57):
    per voxel the mean position and the renormalised sum of the unit normals, as (points, normals) float64."""
    tp = _dev(points)
    if tp is not None:
        tn = _dev(normals)
        tn = tn if tn is not None else _torch().as_tensor(np.ascontiguousarray(normals), device=tp.device)
        p, q = tp, tn
    else:
        p, q = np.ascontiguousarray(points, np.float64), np.ascontiguousarray(normals, np.float64)
    if len(p.shape) != 2 or len(q.shape) != 2 or p.shape[1] != 3 or q.shape[1] != 3:
        raise ValueError("voxel_downsample_with_normals expects Nx3 inputs")
    if p.shape[0] != q.shape[0]:
        raise ValueError("voxel_downsample_with_normals points/normals size mismatch")
    out_p, out_n, _ = _c.voxel_downsample(p, voxel_size, "point_normal", normals=q)
    return out_p, out_n


class DeviceLidarScan:
    """The pixel fields of a LidarScan as CUDA tensors (h x w each, torch, DLPack-exportable); the
    per-column / per-packet headers stay in the host LidarScan `self.host` (they are a few KB and the
    host state machine owns them)."""

    def __init__(self, info, device=0, fused_returns=0, xyz_dtype=np.float32):
        torch = _torch()
        self.info, self.host = info, LidarScan(info)
        self.h, self.w = self.host.h, self.host.w
        dev = torch.device("cuda", device)
        tdt = {np.dtype(np.uint8): torch.uint8, np.dtype(np.uint16): torch.int16, np.dtype(np.uint32): torch.int32,
               np.dtype(np.uint64): torch.int64, np.dtype(np.int8): torch.int8, np.dtype(np.int16): torch.int16,
               np.dtype(np.int32): torch.int32, np.dtype(np.int64): torch.int64,
               np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}
        self._fields = {}
        for name in self.host.fields:
            a = self.host.field(name)
            self._fields[name] = torch.zeros(a.shape, dtype=tdt[a.dtype], device=dev)
        xt = torch.float64 if np.dtype(xyz_dtype) == np.float64 else torch.float32
        self.xyz = [torch.zeros((self.h * self.w, 3), dtype=xt, device=dev) for _ in range(fused_returns)]
        self.range_destaggered = [torch.zeros((self.h, self.w), dtype=torch.int32, device=dev)
                                  for _ in range(fused_returns)]

    @property
    def fields(self):
        return list(self._fields)

    def field(self, name):
        """CUDA tensor of the field (unsigned 16/32-bit fields come as the same-width signed torch dtype:
        identical bits; `.view(torch.uint16)` etc. where torch has the type)."""
        return self._fields[name]

    def field_dtype(self, name):
        """The field's numpy dtype in the reference (e.g. uint16 for a field held in an int16 tensor)."""
        return self.host.field(name).dtype

    # headers, as on LidarScan
    timestamp = property(lambda self: self.host.timestamp)
    measurement_id = property(lambda self: self.host.measurement_id)
    status = property(lambda self: self.host.status)
    packet_timestamp = property(lambda self: self.host.packet_timestamp)
    frame_id = property(lambda self: self.host.frame_id)


class DeviceScanBatcher:
    """ScanBatcher whose decoded scan stays on the GPU: the reference's per-packet state machine
    (lidar_frame.cpp:1698-1959, host) + the fused decode launch writing into the DeviceLidarScan's
    CUDA tensors.  With `lut` the same launch also produces scan.xyz[r] / scan.range_destaggered[r].

        batcher = DeviceScanBatcher(info, lut=XYZLutFloat(info))
        scan = batcher.new_scan()
        for packet, ts in stream:
            if batcher(packet, ts, scan):
                n = normals(destagger(info, scan.xyz[0].reshape(h, w, 3)), scan.range_destaggered[0], origins)
    """

    def __init__(self, info, lut=None, device=0):
        self.info, self.device = info, device
        self._b = FrameBatcher(info)
        self._lut = lut._lut if isinstance(lut, _XYZLutBase) else lut
        if self._lut is not None:
            self._b.set_fused_cloud(self._lut, info.pixel_shift_by_row)
        self._bound = None

    def new_scan(self):
        n_ret = 0
        if self._lut is not None:
            names = LidarScan(self.info).fields
            n_ret = 1 + int("RANGE2" in names)
        return DeviceLidarScan(self.info, self.device, n_ret, self._lut.dtype if self._lut is not None else np.float32)

    def _bind(self, scan):
        if self._bound is not scan:
            self._b.set_device_outputs({n: scan.field(n) for n in scan.fields}, scan.xyz or None,
                                       scan.range_destaggered or None)
            self._bound = scan

    def batch(self, packet, host_timestamp, scan):
        self._bind(scan)
        return self._b.batch(packet, host_timestamp, scan.host)

    __call__ = batch

    def batch_burst(self, packets, host_timestamps, scan):
        self._bind(scan)
        return self._b.batch_burst(packets, host_timestamps, scan.host)

    def flush(self, scan):
        self._bind(scan)
        self._b.flush(scan.host)

    def reset(self):
        self._b.reset()

    batched_packets = property(lambda self: self._b.batched_packets)
    dropped_packets = property(lambda self: self._b.dropped_packets)


# ---- frame-to-map registration (DESIGN f-6) -----------------------------------------------------------
# ouster.sdk.core.VoxelHashMap3d (processing.cpp:395-470, 1040-1055) and ouster.sdk.mapping.ICPRegistration /
# AdaptiveThreshold (python/src/cpp/mapping/_mapping_registration.cpp).  numpy in and out as in the reference; torch
# CUDA tensors are accepted as well and keep the work on the device.

DBL_MAX = _c.DBL_MAX


def _point3(point):
    d = _dev(point)
    p = d.double().reshape(-1) if d is not None else np.ascontiguousarray(point, np.float64).reshape(-1)
    if p.shape[0] != 3:
        raise ValueError("VoxelHashMap method expects a 3-element point")
    return p


def _rows3(points, msg="add_points expects an Nx3 array"):
    d = _dev(points)
    p = d if d is not None else np.ascontiguousarray(points, np.float64)
    if len(p.shape) != 2 or p.shape[1] != 3:
        raise ValueError(msg)
    return p


def _point_xd(point):
    """x, y, z of a (3 + attributes)-element point (VoxelHashMapXd reads the spatial part only)."""
    d = _dev(point)
    p = d.double().reshape(-1) if d is not None else np.ascontiguousarray(point, np.float64).reshape(-1)
    if p.shape[0] < 3:
        raise ValueError("VoxelHashMap method expects a (3+attributes)-element point")
    return p[:3]


class _VoxelHashMap:
    """What VoxelHashMap3d and VoxelHashMapXd share (bind_voxel_hash_map_common, processing.cpp:396-470); the
    subclasses say how a point and a batch of rows are read."""

    @property
    def empty(self):
        return self._m.size()[0] == 0

    def max_points_per_voxel(self):
        return self._m.max_points_per_voxel

    def min_pts_threshold(self):
        return self._m.min_pts_threshold

    def clear(self):
        self._m.clear()

    def add_points(self, points):
        self._m.add_points(self._rows(points))

    def point_cloud(self):
        return self._m.point_cloud()

    def remove_voxels_far_from_location(self, point):
        self._m.remove_far(self._point(point))

    def extract_voxels_far_from_location(self, point):
        return self._m.remove_far(self._point(point), extract=True)

    def get_closest_neighbor(self, point, max_distance_sq=DBL_MAX):
        """(closest point [cols] float64, squared distance); (zeros, max_distance_sq) when nothing qualifies."""
        p = self._point(point)
        nb, d2 = self._m.closest_neighbors(p.reshape(1, 3), max_distance_sq)
        if _c._is_torch(nb):
            nb, d2 = nb.cpu().numpy(), d2.cpu().numpy()
        return nb[0], float(d2[0])


class VoxelHashMap3d(_VoxelHashMap):
    """core.VoxelHashMap3d: first_n_point voxel map, held in device memory.  point_cloud() and
    extract_voxels_far_from_location() list voxels in creation order (the reference: hash-map order, DESIGN 9)."""

    def __init__(self, voxel_size=0.1, max_distance=100.0, max_points_per_voxel=20, min_pts_threshold=1):
        self._m = _c.VoxelMap(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold)

    _point = staticmethod(_point3)
    _rows = staticmethod(_rows3)

    def get_closest_neighbors(self, points, max_distance_sq=DBL_MAX):
        """Batched get_closest_neighbor: (points [n, 3], squared distances [n]); CUDA tensors in, CUDA tensors out."""
        return self._m.closest_neighbors(_rows3(points, "VoxelHashMap method expects a 3-element point"),
                                         max_distance_sq)


class VoxelHashMapXd(_VoxelHashMap):
    """core.VoxelHashMapXd (processing.cpp:1058-1067): the first_n_point map with num_attributes doubles after x, y, z
    in every point, held in device memory (DESIGN f-11).  Voxels, the gate and the searches use x, y, z; rows come out
    3 + num_attributes wide, in creation order."""

    def __init__(self, voxel_size=0.1, max_distance=100.0, max_points_per_voxel=20, min_pts_threshold=1,
                 num_attributes=0):
        self._m = _c.VoxelMap(voxel_size, max_distance, max_points_per_voxel, min_pts_threshold,
                              num_attributes=num_attributes)

    _point = staticmethod(_point_xd)

    def add_points(self, points):
        """Rows of 3 + num_attributes columns; even with no attributes this is the rows call, whose width error is
        the reference's"""
        self._m.add_rows(self._rows(points))

    @staticmethod
    def _rows(points):
        d = _dev(points)
        p = d if d is not None else np.ascontiguousarray(points, np.float64)
        if len(p.shape) != 2 or p.shape[1] < 3:
            raise ValueError("add_points expects at least Nx(3+num_attributes) columns")
        return p

    def get_closest_neighbors(self, points, max_distance_sq=DBL_MAX):
        """Batched get_closest_neighbor on the first three columns of `points`: (rows [n, 3 + num_attributes],
        squared distances [n]); CUDA tensors in, CUDA tensors out."""
        p = self._rows(points)
        return self._m.closest_neighbors(p[:, :3] if _c._is_torch(p) else np.ascontiguousarray(p[:, :3]),
                                         max_distance_sq)


class ICPRegistration:
    """mapping.ICPRegistration(max_num_iterations=50, convergence_criterion=1e-4, max_num_threads=0).
    max_num_threads has no effect on the GPU; like the reference it reads back as a positive number."""

    def __init__(self, max_num_iterations=50, convergence_criterion=0.0001, max_num_threads=0):
        import os
        self.max_num_iterations = int(max_num_iterations)
        self.convergence_criterion = float(convergence_criterion)
        self.max_num_threads = int(max_num_threads) if max_num_threads > 0 else (os.cpu_count() or 1)

    def align_points_to_map(self, frame, voxel_map, max_distance, kernel_scale):
        """4x4 float64 correction that moves `frame` onto the map (a CUDA tensor for a CUDA-tensor frame)."""
        m = voxel_map._m if isinstance(voxel_map, _VoxelHashMap) else voxel_map
        pose, _ = _c.icp_align(m, _rows3(frame), max_distance, kernel_scale, self.max_num_iterations,
                               self.convergence_criterion)
        return pose


def build_linear_system(source, target, kernel_scale):
    """mapping build_linear_system over the pairs (source[i], target[i]): (JtJ 6x6, lower triangle, Jtr [6])."""
    return _c.icp_linear_system(source, target, kernel_scale)


class AdaptiveThreshold:
    """mapping.AdaptiveThreshold (adaptive_threshold.h, adaptive_threshold.cpp): host scalars."""

    def __init__(self, max_range, initial_threshold=2.0, min_motion_threshold=0.01):
        self.min_motion_threshold = float(min_motion_threshold)
        self.max_range = float(max_range)
        self.model_sse = float(initial_threshold) * float(initial_threshold)
        self.num_samples = 1

    @staticmethod
    def _angle(r):
        """Eigen::AngleAxisd(R).angle(): R -> quaternion (Quaternion.h, quaternionbase_assign_impl), then
        2 atan2(|vec|, |w|)."""
        t = r[0, 0] + r[1, 1] + r[2, 2]
        if t > 0:
            s = np.sqrt(t + 1.0)
            w = 0.5 * s
            s = 0.5 / s
            v = np.array([(r[2, 1] - r[1, 2]) * s, (r[0, 2] - r[2, 0]) * s, (r[1, 0] - r[0, 1]) * s])
        else:
            i = 0
            if r[1, 1] > r[0, 0]:
                i = 1
            if r[2, 2] > r[i, i]:
                i = 2
            j, k = (i + 1) % 3, (i + 2) % 3
            s = np.sqrt(r[i, i] - r[j, j] - r[k, k] + 1.0)
            v = np.zeros(3)
            v[i] = 0.5 * s
            s = 0.5 / s
            w = (r[k, j] - r[j, k]) * s
            v[j] = (r[j, i] + r[i, j]) * s
            v[k] = (r[k, i] + r[i, k]) * s
        n = float(np.linalg.norm(v))
        return 0.0 if n < np.finfo(np.float64).eps else 2.0 * np.arctan2(n, abs(w))

    def update_model_deviation(self, current_deviation):
        m = np.asarray(current_deviation, np.float64).reshape(4, 4)
        delta_rot = 2.0 * self.max_range * np.sin(self._angle(m[:3, :3]) / 2.0)
        delta_trans = float(np.linalg.norm(m[:3, 3]))
        model_error = delta_trans + delta_rot
        if model_error > self.min_motion_threshold:
            self.model_sse += model_error * model_error
            self.num_samples += 1

    def compute_threshold(self):
        return float(np.sqrt(self.model_sse / self.num_samples))


# ---- cloud-to-cloud ICP (DESIGN f-7) ------------------------------------------------------------------
# ouster.sdk.algorithm.point_to_point_align / point_to_plane_align (python/src/cpp/_algorithm.cpp:158-245): numpy in,
# a (4, 4) float64 numpy array out, as in the reference; CUDA tensors in give a CUDA tensor out with no host wait.

def _interp_pose(x_interp, x_known, poses_known, pose_dtype):
    """processing.cpp:241-338: shapes (N,) or (N, 1), x as float64, poses (M, 4, 4) converted to pose_dtype."""
    def xshape(a, name):
        if len(a.shape) != 1 and (len(a.shape) != 2 or a.shape[1] != 1):
            raise RuntimeError(f"{name} must have shape (N,) or (N,1)")
    xshape(x_interp, "x_interp")
    xshape(x_known, "x_known")
    if len(poses_known.shape) != 3 or tuple(poses_known.shape[1:]) != (4, 4):
        raise RuntimeError("poses_known must have shape (M, 4, 4)")
    if x_known.shape[0] != poses_known.shape[0]:
        raise RuntimeError("The number of poses in poses_known must match the number of values in x_known")
    if x_known.shape[0] < 2:
        raise ValueError("Not enough evaluation poses for interpolation")
    if _c._is_torch(x_interp):
        torch = _torch()
        tdt = torch.float64 if pose_dtype == np.float64 else torch.float32
        x, k = x_interp.to(torch.float64), x_known.to(x_interp.device, torch.float64)
        pk = poses_known.to(x_interp.device, tdt)
    else:
        x, k = np.asarray(x_interp, np.float64), np.asarray(x_known, np.float64)
        pk = np.asarray(poses_known, pose_dtype)
    return _c.interp_pose(x, k, pk)


def interp_pose(x_interp, x_known, poses_known):
    """Interpolate 4x4 poses at x_interp (float64): (N, 4, 4) float64 (processing.cpp:1017-1027).  numpy in and out,
    or CUDA tensors on their device."""
    return _interp_pose(x_interp, x_known, poses_known, np.float64)


def interp_pose_float(x_interp, x_known, poses_known):
    """interp_pose with float32 poses: known poses widened, each result rounded once (processing.cpp:1029-1039)."""
    return _interp_pose(x_interp, x_known, poses_known, np.float32)


class DeskewMethod:
    """mapping::DeskewMethod (deskew_method.h, _mapping_slam.cpp:238-270): keeps the last two registered poses."""

    def __init__(self, infos, initial_pose=None):
        if len(infos) == 0:
            raise ValueError("No sensor info provided for slam")
        self._ts, self._poses = [], []
        self._initial = np.eye(4) if initial_pose is None else np.array(initial_pose, np.float64).reshape(4, 4)

    def set_last_pose(self, ts, pose):
        pose = np.asarray(pose, np.float64)
        if pose.shape != (4, 4):
            raise RuntimeError("pose must be a (4,4) array representing a transformation matrix")
        if len(self._ts) >= 2:
            self._ts.pop(0)
            self._poses.pop(0)
        self._ts.append(int(ts) * 1e-9)
        self._poses.append(pose.copy())

    def finalize_after_registration(self, frames, anchor_timestamp_ns, corrected_anchor_pose):
        self.set_last_pose(anchor_timestamp_ns, corrected_anchor_pose)

    def update(self, frames):
        raise NotImplementedError


class ConstantVelocityDeskewMethod(DeskewMethod):
    """ConstantVelocityDeskewMethod::update (deskew_method.cpp:55-71): every valid column of every frame gets the
    pose at its timestamp on the motion through the last two poses, or the initial pose before there are two.
    `frames`: a list with None for empty slots, of LidarScan or DeviceLidarScan (whose poses are host-side).
    One ob_frames_interp_pose call for the whole set."""

    def update(self, frames):
        items = []
        for f in frames:
            if f is None:
                items.append(None)
                continue
            host = f.host if isinstance(f, DeviceLidarScan) else f
            items.append((host.timestamp, host.status, host.body_to_world))
        if len(self._ts) < 2:
            _c.frames_interp_pose(items, 0.0, self._initial)
        else:
            _c.frames_interp_pose(items, self._ts[0], self._poses[0], self._ts[-1], self._poses[-1])
        return frames


def _return_field_name(base, ret):
    """ChanField::return_field_name: `base` for return 0, then base + "2", base + "3", ..."""
    return base if ret <= 0 else base + str(ret + 1)


class GroundSegConfig:
    """GroundSegConfig (ground_seg.h): grid_size, the cell size in metres of the 2.5-D height map."""

    def __init__(self, grid_size=0.5):
        self.grid_size = grid_size


class GroundSegEngine:
    """GroundSegEngine (ground_seg.cpp:1346-1416).  update(frames) segments the frames of a set in one
    ob_ground_mask call: `frames` is a list with None for empty slots, of LidarScan or DeviceLidarScan.  Each frame
    gets GROUND (and GROUND2, ... up to its sensor's returns) as uint8 pixel fields, deleted and re-added zeroed,
    then filled where the frame keeps its pixels (host arrays, or device tensors); GROUND fields beyond the returns
    the frame has (up to the first missing RANGEk) are removed.  A frame without float32 NORMALS gets the normals
    the reference computes, with the sensor's sensor_to_body.  A DeviceLidarScan's poses and status are read from
    its host side.  One LUT (with extrinsics) is kept per sensor serial number.  Returns `frames`."""

    def __init__(self, config):
        self.config = config
        self._luts = {}

    @staticmethod
    def create(config=None):
        config = GroundSegConfig() if config is None else config
        g = float(config.grid_size)
        if not np.isfinite(g) or g <= 0.0:
            raise ValueError("GroundSegConfig.grid_size must be > 0")
        return GroundSegEngine(config)

    def _lut(self, info):
        key = getattr(info, "sn", 0)
        if key not in self._luts:
            self._luts[key] = XYZLut(info, use_extrinsics=True)._lut
        return self._luts[key]

    def update(self, frames):
        items, plans = [], []
        for f in frames:
            if f is None:
                items.append(None)
                continue
            dev = isinstance(f, DeviceLidarScan)
            info = f.info if dev else f.sensor_info
            if info is None:
                raise ValueError("frame.sensor_info is required for get_ground_mask")
            names = f.fields
            if ChanField.RANGE not in names:
                raise ValueError("frame must contain RANGE field for get_ground_mask")
            n_max = 2 if "DUAL" in str(getattr(info, "profile", "")).upper() else 1
            ranges = [f.field(ChanField.RANGE)]
            for ret in range(1, n_max):
                name = _return_field_name(ChanField.RANGE, ret)
                if name not in names:
                    break
                ranges.append(f.field(name))
            masks = []
            for ret in range(n_max):
                name = _return_field_name(ChanField.GROUND, ret)
                if dev:
                    f._fields[name] = _torch().zeros((f.h, f.w), dtype=_torch().uint8, device=ranges[0].device)
                    masks.append(f._fields[name])
                else:
                    if name in names:
                        f.del_field(name)
                    f.add_field(name, np.uint8)
                    masks.append(f.field(name))
            host = f.host if dev else f
            item = {"lut": self._lut(info), "ranges": ranges, "status": host.status, "poses": host.body_to_world,
                    "masks": masks[:len(ranges)]}
            nrm = [f.field(k) if k in names else None for k in (ChanField.NORMALS, ChanField.NORMALS2)]
            if nrm[0] is not None and str(nrm[0].dtype) in ("float32", "torch.float32"):
                item["normals"] = nrm[0]
                if nrm[1] is not None and len(ranges) > 1:
                    item["normals2"] = nrm[1]
            else:
                s2b = getattr(info, "sensor_to_body", None)
                item["sensor_to_body"] = np.eye(4) if s2b is None else np.asarray(s2b, np.float64)
            items.append(item)
            plans.append((f, dev, len(ranges), n_max))
        _c.ground_mask(items, grid_size=self.config.grid_size)
        for f, dev, n_found, n_max in plans:
            for ret in range(n_found, n_max):
                name = _return_field_name(ChanField.GROUND, ret)
                if dev:
                    f._fields.pop(name, None)
                elif name in f.fields:
                    f.del_field(name)
        return frames


def _imu_measurements_per_frame(info):
    """format.imu_measurements_per_packet * format.imu_packets_per_frame (deskew_method.cpp:800-801) of a sensor
    info object or metadata dict; 0 when the info has no format."""
    fmt = _sensor_value(info, "format")
    if fmt is None:
        return 0
    return int(_sensor_value(fmt, "imu_measurements_per_packet", 0) or 0) * \
        int(_sensor_value(fmt, "imu_packets_per_frame", 0) or 0)


class DeskewMethodFactory:
    """DeskewMethodFactory::create (deskew_method.cpp:790-832).  IMU packets are not decoded in this project, so
    "imu_deskew", and "auto" when a sensor reports IMU measurements, raise instead of deskewing (DESIGN 9)."""

    @staticmethod
    def create(method_name, infos):
        if method_name == "none":
            return None
        if method_name == "constant_velocity":
            return ConstantVelocityDeskewMethod(infos)
        imu_text = "IMU deskew is not supported: IMU packets are not decoded"
        if method_name == "imu_deskew":
            raise ValueError(imu_text)
        if method_name == "auto":
            if any(_imu_measurements_per_frame(i) > 0 for i in infos):
                raise ValueError(imu_text)
            return ConstantVelocityDeskewMethod(infos)
        raise ValueError("Invalid deskew_method: " + method_name)


def point_to_point_align(source_points, target_points, initial_guess=None, max_corr_dist=0.25):
    """source_to_target_transform by point-to-point ICP with MAD-scaled Huber weights (at most 10 iterations);
    initial_guess (identity when None) comes back when fewer than 20 usable points or correspondences exist."""
    pose, _ = _c.cloud_align(_rows3(source_points, "source_points must be Nx3"),
                             _rows3(target_points, "target_points must be Nx3"),
                             initial_guess=initial_guess, max_corr_dist=max_corr_dist)
    return pose


def point_to_plane_align(source_points, target_points, source_normals, target_normals, initial_guess=None,
                         max_corr_dist=0.25, max_normal_angle_deg=20.0):
    """source_to_target_transform by point-to-plane ICP: correspondences whose normals differ by more than
    max_normal_angle_deg are rejected, non-finite points and normals are ignored, normals are normalised."""
    pose, _ = _c.cloud_align(_rows3(source_points, "source_points must be Nx3"),
                             _rows3(target_points, "target_points must be Nx3"),
                             _rows3(source_normals, "source_normals must be Nx3"),
                             _rows3(target_normals, "target_normals must be Nx3"),
                             initial_guess=initial_guess, max_corr_dist=max_corr_dist,
                             max_normal_angle_deg=max_normal_angle_deg)
    return pose


def align_clouds(*args, initial_guess=None, compute_confidence=False):
    """source_to_target_transform between two point clouds without a usable initial guess (DESIGN f-14):
    align_clouds(source_points, target_points, initial_guess=None, compute_confidence=False) or
    align_clouds(source_points, source_normals, target_points, target_normals, initial_guess=None,
    compute_confidence=False), dispatched on the number of arrays as the reference's two bindings are.  A yaw search
    by BEV cross-correlation, three ICP passes, and the overlap confidence as a guard.  Returns the 4x4 pose, or
    (pose, confidence) with compute_confidence."""
    # (sp, tp, initial_guess, compute_confidence) has a flag where (sp, sn, tp, tn) has an array
    n_arrays = 4 if len(args) >= 4 and getattr(args[3], "ndim", np.ndim(args[3])) >= 1 else 2
    if len(args) < 2 or len(args) > n_arrays + 2:
        raise TypeError("align_clouds() takes 2 or 4 point arrays, then initial_guess and compute_confidence")
    rest = list(args[n_arrays:])
    if rest:
        initial_guess = rest.pop(0)
    if rest:
        compute_confidence = rest.pop(0)
    if n_arrays == 4:
        sp, sn, tp, tn = args[:4]
    else:
        (sp, tp), sn, tn = args[:2], None, None
    pose, conf = _c.align_clouds(sp, tp, sn, tn, initial_guess=initial_guess,
                                 compute_confidence=compute_confidence)
    return (pose, conf) if compute_confidence else pose


# ---- zone monitoring (DESIGN f-8)-----------------------------------------------------------------------------
# ouster.sdk.core's Mesh / Stl / Zone / ZoneSet / Zrb (python/src/cpp/client/zone_monitor.cpp) and EmulatedZoneMon
# (python/src/ouster/sdk/core/zone_common.py).  Rendering and the per-frame occupancy run on the GPU; STL parsing
# is host code.  ZRB / ZoneSet files, hashes and JSON are not provided (DESIGN 9).
import re as _re  # noqa: E402
from fractions import Fraction as _Fraction  # noqa: E402
import struct as _struct  # noqa: E402
import sys as _sys  # noqa: E402

MAX_ACTIVE_ZONES = 16
MAX_AVAILABLE_ZONES = 128


class CoordinateFrame(enum.IntEnum):
    NONE = 0
    BODY = 1
    SENSOR = 2


class ZoneMode(enum.IntEnum):
    NONE = 0
    OCCUPANCY = 1
    VACANCY = 2


_STL_HEADER_BYTES = 80
_NUM = rb"(-?[0-9\.]+(?:[eE][+-]\d+)?)"
_VERTEX_RE = _re.compile(rb"^\s*vertex\s+" + _NUM + rb"\s+" + _NUM + rb"\s+" + _NUM, _re.ASCII)
_STOF_RE = _re.compile(rb"[+-]?(?:\d+\.?\d*|\.\d+)(?:[eE][+-]?\d+)?", _re.ASCII)


def _stl_error(message, line=b""):
    """mesh.cpp:86-92"""
    msg = "STL Parsing Error: " + message
    if line:
        msg += ": '" + line.decode("latin-1") + "'"
    print(msg, file=_sys.stderr)


_FLT_MIN = _Fraction(2) ** -126
_FLT_INF_EDGE = _Fraction(2) ** 128 - _Fraction(2) ** 103  # halfway between FLT_MAX and 2^128


def _stof(s):
    """std::stof on a token the vertex regex accepted: strtof's longest numeric prefix, rounded once to the nearest
    float (ties to even).  No prefix, or a result strtof flags with ERANGE (overflow, or a nonzero value that ends
    up subnormal or zero), raises ValueError, where std::stof throws."""
    m = _STOF_RE.match(s)
    if not m:
        raise ValueError("stof: no conversion")
    q = _Fraction(m.group(0).decode())
    if abs(q) >= _FLT_INF_EDGE:
        raise ValueError("stof: out of range")
    if q == 0:
        return np.float32(-0.0) if m.group(0)[:1] == b"-" else np.float32(0.0)
    # float(q) rounds once to double; rounding that to float can land one step off, so pick the nearest neighbour
    f = np.float32(float(q))
    with np.errstate(over="ignore"):
        cands = [c for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf)))
                 if np.isfinite(c)]
    best = min(cands, key=lambda c: (abs(_Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1))
    if abs(_Fraction(float(best))) < _FLT_MIN and _Fraction(float(best)) != q:
        raise ValueError("stof: out of range")
    return np.float32(best)


def _ascii_lines(data):
    """read_stl_ascii_line (mesh.cpp:73-84): trimmed of ' \\t\\r', blank and '#' lines skipped, lower-cased"""
    for raw in data.split(b"\n"):
        line = raw.strip(b" \t\r")
        if not line or line[:1] == b"#":
            continue
        yield line.lower()


def _load_stl_ascii(data):
    """Mesh::load_from_stl_ascii, mesh.cpp:94-173: (n, 3, 3) float32 or None"""
    lines = _ascii_lines(data)
    line = next(lines, None)
    if line is None or not _re.search(rb"^\s*solid\b", line):
        _stl_error("Failed to find 'solid' header", line or b"")
        return None
    tris = []
    for line in lines:
        if _re.search(rb"^\s*facet\b", line):
            line = next(lines, None)
            if line is None or not _re.search(rb"^\s*outer\s+loop", line):
                _stl_error("Expected 'outer loop'", line or b"")
                return None
            verts = []
            for _ in range(3):
                line = next(lines, None)
                m = _VERTEX_RE.search(line) if line is not None else None
                if m is None:
                    _stl_error("Expected 'vertex'", line or b"")
                    return None
                verts.append([_stof(m.group(k)) for k in (1, 2, 3)])
            for word in (b"endloop", b"endfacet"):
                line = next(lines, None)
                if line is None or not _re.search(rb"^\s*" + word, line):
                    _stl_error(f"Expected '{word.decode()}'", line or b"")
                    return None
            tris.append(verts)
        elif _re.search(rb"^\s*endsolid\b", line):
            return np.array(tris, np.float32).reshape(-1, 3, 3)
        else:
            _stl_error("Unexpected line outside of a facet", line)
            return None
    _stl_error("File ended unexpectedly without 'endsolid'")
    return None


def _load_stl_binary(data):
    """Mesh::load_from_stl_binary, mesh.cpp:175-207: 80-byte header, uint32 count, then 50-byte records (a
    normal and three vertices, 12 floats, and a 2-byte attribute count that may be cut short at the end)"""
    if len(data) < _STL_HEADER_BYTES:
        _stl_error("File too short.")
        return None
    if len(data) < _STL_HEADER_BYTES + 4:
        _stl_error("Unknown # of n_tris.")
        return None
    n = _struct.unpack_from("<I", data, _STL_HEADER_BYTES)[0]
    if n and len(data) < 84 + 50 * (n - 1) + 48:
        _stl_error("Mismatch in # of n_tris.")
        return None
    rec = np.dtype([("normal", "<f4", 3), ("v", "<f4", (3, 3)), ("attr", "<u2")])
    full = min(n, (len(data) - 84) // 50)
    tris = np.frombuffer(data, rec, full, 84)["v"] if full else np.zeros((0, 3, 3), np.float32)
    if full < n:  # the last record without its attribute bytes
        tail = np.frombuffer(data, "<f4", 12, 84 + 50 * full)[3:].reshape(1, 3, 3)
        tris = np.concatenate([tris, tail])
    return np.ascontiguousarray(tris, np.float32)


def load_stl_triangles(data):
    """Mesh::load_from_stl_bytes (mesh.cpp:209-241): ASCII when "endsolid" (any case) starts after the 80-byte
    header, else binary.  -> (n, 3, 3) float32 vertices, or None where the reference returns false."""
    pos = bytes(data).lower().find(b"endsolid")
    if pos > _STL_HEADER_BYTES:
        return _load_stl_ascii(bytes(data))
    return _load_stl_binary(bytes(data))


class Mesh:
    """Mesh (mesh.h): the triangles of an STL as an (n, 3, 3) float32 array."""

    def __init__(self, triangles=None):
        self._t = np.zeros((0, 3, 3), np.float32) if triangles is None else \
            np.ascontiguousarray(triangles, np.float32).reshape(-1, 3, 3)

    @property
    def triangles(self):
        return self._t

    def load_from_stl_bytes(self, data):
        t = load_stl_triangles(data)
        if t is None:
            return False
        self._t = t
        return True

    def load_from_stl(self, path):
        with open(path, "rb") as f:
            return self.load_from_stl_bytes(f.read())


class Stl:
    """Stl (stl.h): the file's bytes and the zone's coordinate frame."""

    def __init__(self, path_or_bytes):
        if isinstance(path_or_bytes, (bytes, bytearray)):
            self.blob = bytes(path_or_bytes)
        else:
            with open(path_or_bytes, "rb") as f:
                self.blob = f.read()
        self.coordinate_frame = CoordinateFrame.NONE

    def to_mesh(self):
        m = Mesh()
        if not m.load_from_stl_bytes(self.blob):
            raise RuntimeError("Stl: failed to parse STL")
        return m


class Zrb:
    """Zrb (zrb.h): near / far range images in mm and the transforms they were rendered with."""

    def __init__(self, near_range_mm=None, far_range_mm=None, serial_number=0, beam_to_lidar_transform=None,
                 lidar_to_sensor_transform=None, sensor_to_body_transform=None):
        self.near_range_mm = np.zeros((0, 0), np.uint32) if near_range_mm is None else near_range_mm
        self.far_range_mm = np.zeros((0, 0), np.uint32) if far_range_mm is None else far_range_mm
        self.serial_number = serial_number
        self.beam_to_lidar_transform = np.eye(4) if beam_to_lidar_transform is None else beam_to_lidar_transform
        self.lidar_to_sensor_transform = np.eye(4) if lidar_to_sensor_transform is None else lidar_to_sensor_transform
        self.sensor_to_body_transform = np.eye(4) if sensor_to_body_transform is None else sensor_to_body_transform
        self.stl_hash = None


def _sensor_value(info, key, default=None):
    return info.get(key, default) if isinstance(info, dict) else getattr(info, key, default)


class BeamConfig:
    """BeamConfig (beam_config.cpp:23-52): the sensor's beams and the two LUTs zones are rendered with, built on
    the GPU in float64 (range unit 0.001; the BODY LUT uses scale_translation(sensor_to_body) * lidar_to_sensor)."""

    def __init__(self, n_cols, px_altitudes, px_azimuths, beam_to_lidar_transform, lidar_to_sensor_transform,
                 sensor_to_body_transform=None, m_per_zmbin=0.0074927621875, serial_number=0, device=0):
        self.n_cols, self.n_rows = int(n_cols), len(px_altitudes)
        self.beam_to_lidar_transform = np.array(beam_to_lidar_transform, np.float64).reshape(4, 4)
        self.lidar_to_sensor_transform = np.array(lidar_to_sensor_transform, np.float64).reshape(4, 4)
        self.sensor_to_body_transform = None if sensor_to_body_transform is None else \
            np.array(sensor_to_body_transform, np.float64).reshape(4, 4)
        self.m_per_zmbin, self.serial_number = m_per_zmbin, serial_number
        self.px_altitudes, self.px_azimuths = list(px_altitudes), list(px_azimuths)
        if not self.beam_to_lidar_transform.any():
            raise RuntimeError("BeamConfig: beam_to_lidar_transform not set")
        if not self.lidar_to_sensor_transform.any():
            raise RuntimeError("BeamConfig: lidar_to_sensor_transform not set")
        lut = lambda tr: _c.XYZLutT.from_intrinsics(self.n_cols, self.n_rows, 0.001, self.beam_to_lidar_transform,
                                                    tr, self.px_azimuths, self.px_altitudes, np.float64, device)
        self.lut_no_sensor_to_body_transform = lut(self.lidar_to_sensor_transform)
        self.lut = None
        if self.sensor_to_body_transform is not None:
            s2b = self.sensor_to_body_transform.copy()
            s2b[:3, 3] *= 1000
            self.lut = lut(s2b @ self.lidar_to_sensor_transform)

    @classmethod
    def from_sensor_info(cls, info, sensor_to_body_transform=None, device=0):
        return cls(_sensor_value(info, "w"), _sensor_value(info, "beam_altitude_angles"),
                   _sensor_value(info, "beam_azimuth_angles"), _sensor_value(info, "beam_to_lidar_transform"),
                   _sensor_value(info, "lidar_to_sensor_transform"), sensor_to_body_transform,
                   serial_number=_sensor_value(info, "sn", 0), device=device)


class Zone:
    """Zone (zone.h).  render() runs on the GPU."""
    MAX_TRIANGLES = 2048

    def __init__(self):
        self.point_count, self.frame_count, self.mode = 0, 0, ZoneMode.NONE
        self.stl, self.zrb = None, None

    def check_invariants(self):
        """zone.cpp:18-46"""
        if self.point_count == 0:
            raise RuntimeError("Zone: point_count must be in [1, 262143]")
        if self.frame_count == 0:
            raise RuntimeError("Zone: frame_count must be in [1, 65535]")
        if self.stl is None and self.zrb is None:
            raise RuntimeError("Zone: must have either STL or ZRB")
        if self.mode not in (ZoneMode.OCCUPANCY, ZoneMode.VACANCY):
            raise RuntimeError("Zone: mode must be OCCUPANCY or VACANCY")
        if self.stl is not None:
            if not self.stl.blob:
                raise RuntimeError("Zone: STL blob cannot be empty")
            if self.stl.coordinate_frame == CoordinateFrame.NONE:
                raise RuntimeError("Zone: STL coordinate frame must be BODY or SENSOR")
        if self.zrb is not None and np.count_nonzero(self.zrb.far_range_mm != 0) < self.point_count:
            raise RuntimeError("Zone: ZRB far range image has fewer nonzero pixels than point_count")

    def _renderable(self, config):
        """The early returns of Zone::render (zone.cpp:64-85): the mesh, or None after the reference's message."""
        self.check_invariants()
        if self.stl is None:
            print("Zone: Error rendering zone, no STL provided.", file=_sys.stderr)
            return None
        tris = self.stl.to_mesh().triangles
        if len(tris) == 0:
            print("Zone: Error rendering zone, STL has no triangles.", file=_sys.stderr)
            return None
        if len(tris) > self.MAX_TRIANGLES:
            print("Zone: Error rendering zone, STL has too many triangles.", file=_sys.stderr)
            return None
        if self.stl.coordinate_frame == CoordinateFrame.BODY and config.sensor_to_body_transform is None:
            print("Zone: Error rendering zone, sensor_to_body_transform not set for BODY coordinate frame.",
                  file=_sys.stderr)
            return None
        return tris

    def render(self, config):
        """Zone::render(BeamConfig): True with self.zrb set, False where the reference returns false."""
        return _render_zones([self], config)[0]


def _render_zones(zones, config):
    """Zone::render for several zones in one launch; -> list of bools"""
    todo, meshes = [], []
    ok = [False] * len(zones)
    for i, z in enumerate(zones):
        tris = z._renderable(config)
        if tris is not None:
            todo.append(i)
            meshes.append({"triangles": tris, "coordinate_frame": int(z.stl.coordinate_frame),
                           "point_count": z.point_count, "frame_count": z.frame_count, "mode": int(z.mode)})
    if not todo:
        return ok
    try:
        near, far, px = _c.zone_render(meshes, config.n_rows, config.n_cols, config.lut_no_sensor_to_body_transform,
                                       config.lut, device_out=False)
    except _c._capi.OusterB200Error as e:
        raise RuntimeError(str(e).split("] ", 1)[-1]) from None
    s2b = config.sensor_to_body_transform if config.sensor_to_body_transform is not None else np.eye(4)
    for k, i in enumerate(todo):
        zones[i].zrb = Zrb(near[k], far[k], config.serial_number, config.beam_to_lidar_transform.copy(),
                           config.lidar_to_sensor_transform.copy(), s2b.copy())
        ok[i] = bool(px[k] > 0)
    return ok


class ZoneSet:
    """A minimal ZoneSet (zone_monitor.h): zones by id, power_on_live_ids and sensor_to_body_transform."""

    def __init__(self):
        self.zones = {}
        self.power_on_live_ids = []
        self.sensor_to_body_transform = None

    def render(self, sensor_info, device=0):
        """ZoneSet::render (zone_monitor.cpp:399-448): every zone with an STL, in one GPU launch."""
        config = BeamConfig.from_sensor_info(sensor_info, self.sensor_to_body_transform, device)
        ids = [i for i, z in self.zones.items() if not (z.zrb is not None and z.stl is None)]
        ok = _render_zones([self.zones[i] for i in ids], config)
        for i, good in zip(ids, ok):
            if not good:
                raise RuntimeError(f"ZoneSet::render: zone {i} was out of sensor FOV.")
            self.zones[i].zrb.serial_number = _sensor_value(sensor_info, "sn", 0)


class EmulatedZoneMon:
    """EmulatedZoneMon (zone_common.py:14-136) over a device-resident ZoneMonitor.  calc_triggers takes numpy or
    CUDA range images; with CUDA input nothing waits for the GPU until an attribute or get_packet() is read."""

    def __init__(self, zone_set, device=0):
        if not zone_set.zones:
            raise ValueError("ZoneSet must have at least one zone defined")
        if not all(zone.zrb is not None for zone in zone_set.zones.values()):
            raise ValueError("EmulatedZoneMon: all zones in ZoneSet must have a valid ZRB")
        self.zone_set, self.device = zone_set, device
        self._counts = ({}, {}, {}, {}, {}, {})
        self._triggers = [0] * MAX_AVAILABLE_ZONES
        self._alerts = [0] * MAX_AVAILABLE_ZONES
        self.update_count = 0
        self.rendered_zones = {}
        self.live_zones = list(zone_set.power_on_live_ids)
        self.debug = False
        self.max_counts = {}
        for zone_id, zone in zone_set.zones.items():
            self.max_counts[zone_id] = int(np.count_nonzero(np.asarray(zone.zrb.near_range_mm) <
                                                            np.asarray(zone.zrb.far_range_mm)))
            self.rendered_zones[zone_id] = zone.zrb
        self._mon = None
        self._dirty = False

    def _monitor(self, h, w):
        if self._mon is None or (self._mon.h, self._mon.w) != (h, w):
            if len(self.live_zones) > MAX_ACTIVE_ZONES:
                raise ValueError("at most 16 live zones")
            live = []
            for zone_id in self.live_zones:
                z, zrb = self.zone_set.zones[zone_id], self.rendered_zones[zone_id]
                live.append({"id": zone_id, "mode": int(z.mode), "point_count": z.point_count,
                             "frame_count": z.frame_count, "near_mm": zrb.near_range_mm, "far_mm": zrb.far_range_mm,
                             "triggers": self._triggers[zone_id], "alerts": self._alerts[zone_id]})
            self._mon = _c.ZoneMonitor(live, h, w, self.device)
        return self._mon

    def set_live_zones(self, live_zones):
        self._pull()
        self.live_zones = list(live_zones)
        self._mon = None

    def calc_triggers(self, range_field, bitmask_field=None):
        t = _dev(range_field)
        r = t if t is not None else np.ascontiguousarray(range_field, np.uint32)
        h, w = int(r.shape[0]), int(r.shape[1])
        b = None
        if bitmask_field is not None:
            b = _dev(bitmask_field)
            if b is None:
                b = bitmask_field
                if not isinstance(b, np.ndarray) or b.dtype != np.uint32 or not b.flags["C_CONTIGUOUS"]:
                    raise ValueError("bitmask_field must be a C-contiguous uint32 array")
        self._monitor(h, w).update(r, b)
        self._dirty = True
        if t is None:
            self._pull()

    def _pull(self):
        """read the last update's records and counters back into the reference's attributes"""
        if not self._dirty:
            return
        self._dirty = False
        st = self._mon.states()
        trig, alerts, sums = self._mon.counters()
        dicts = ({}, {}, {}, {}, {}, {})
        keys = ("count", "occlusion_count", "invalid_count", "min_range", "max_range")
        for slot, zone_id in enumerate(self.live_zones):
            for d, k in zip(dicts, keys):
                d[zone_id] = int(st[slot][k])
            # np.mean of the triggering uint32 ranges: their sum is exact in float64 below 2^53, then one division
            cnt = int(st[slot]["count"])
            dicts[5][zone_id] = np.float64(sums[slot]) / cnt if cnt else 0
            self._triggers[zone_id], self._alerts[zone_id] = trig[slot], alerts[slot]
        self._counts = dicts

    def _get(i):
        return property(lambda self: (self._pull(), self._counts[i])[1])

    zone_counts, occlusion_counts, invalid_counts = _get(0), _get(1), _get(2)
    zone_mins, zone_maxes, zone_avgs = _get(3), _get(4), _get(5)
    del _get
    zone_triggers = property(lambda self: (self._pull(), self._triggers)[1])
    zone_alerts = property(lambda self: (self._pull(), self._alerts)[1])

    @property
    def triggered_zone_ids(self):
        return [zone_id for zone_id, alerts in enumerate(self.zone_alerts) if alerts > 0]

    def get_packet(self):
        """the 16 ZoneState records (recarray; id 255 for unused slots)"""
        if self._mon is None:
            zmu = np.zeros(MAX_ACTIVE_ZONES, _c.ZONE_STATE_DTYPE)
            zmu["id"][len(self.live_zones):] = 255
            return zmu.view(np.recarray)
        self._pull()
        return self._mon.states().view(np.recarray)


# ---- image post-processing (ouster.sdk.core.AutoExposure & co., processing.cpp:785-880) -------------------------
# numpy float32 / float64 images are updated in place and the call returns None; a float16 H x W x 3 image returns a
# new float32 array.  Torch CUDA tensors (or device DLPack exporters) are processed in place on the torch current
# stream without waiting for the GPU; the processor's state stays on the device between calls.

def _image_arg(image, allowed):
    """(array, kind) for an update() argument: kind "f16" or "float"; TypeError as nanobind's overload resolution
    raises it for any other dtype or a non-C-contiguous array"""
    d = _dev(image)
    if d is not None:
        torch = _torch()
        kinds = {torch.float16: "f16", torch.float32: "float", torch.float64: "float"}
        ok = d.dtype in kinds and kinds[d.dtype] in allowed and d.is_contiguous()
        a, k = d, kinds.get(d.dtype)
    else:
        a = image
        kinds = {np.dtype(np.float16): "f16", np.dtype(np.float32): "float", np.dtype(np.float64): "float"}
        ok = isinstance(a, np.ndarray) and a.dtype in kinds and kinds[a.dtype] in allowed and a.flags["C_CONTIGUOUS"]
        k = kinds.get(a.dtype) if isinstance(a, np.ndarray) else None
    if not ok:
        raise TypeError("update(): incompatible function arguments")
    return a, k


class _ImageProc:
    _kind = None
    _allowed = ()

    def __init__(self, **kw):
        self._p = _c.ImageProcessor(self._kind, **kw)

    def update(self, image, update_state=True):
        a, k = _image_arg(image, self._allowed)
        if k == "f16" or a.ndim == 3:
            if a.ndim != 3 or a.shape[2] != 3:
                raise ValueError("Expected an H x W x 3 array")
            if self._mono_only:
                raise TypeError("update(): incompatible function arguments")
        elif a.ndim != 2 or self._rgb_only:
            raise TypeError("update(): incompatible function arguments")
        return self._p.update(a, update_state=bool(update_state))

    def _state(self):
        return self._p.state()


class AutoExposure(_ImageProc):
    """AutoExposure(), AutoExposure(update_every), AutoExposure(lo_percentile, hi_percentile, update_every,
    damping=0.9): mono and RGB float32 / float64 in place, float16 RGB to a new float32 array"""
    _kind, _allowed, _mono_only, _rgb_only = "auto_exposure", ("f16", "float"), False, False

    def __init__(self, *args, **kw):
        names = ("lo_percentile", "hi_percentile", "update_every", "damping")
        kw.update(zip(names[2:] if len(args) == 1 else names, args))
        if len(args) not in (0, 1, 3, 4):
            raise TypeError("__init__(): incompatible function arguments")
        kw.setdefault("update_every", 3)
        super().__init__(**kw)


class BeamUniformityCorrector(_ImageProc):
    """BeamUniformityCorrector(): mono float32 / float64 in place"""
    _kind, _allowed, _mono_only, _rgb_only = "beam_uniformity", ("float",), True, False

    def __init__(self):
        super().__init__()


class LocalToneMapper(_ImageProc):
    """LocalToneMapper(), LocalToneMapper(update_every), LocalToneMapper(lo, hi, update_every, damping,
    compress_dr_max_lum | compress_dr, color_correct): float16 RGB to a new float32 array, as the Python binding
    takes it"""
    _kind, _allowed, _mono_only, _rgb_only = "local_tone_map", ("f16",), False, True

    def __init__(self, *args, **kw):
        names = ("lo_percentile", "hi_percentile", "update_every", "damping", "compress_dr_max_lum", "color_correct")
        if "compress_dr" in kw:
            kw["compress_dr_max_lum"] = kw.pop("compress_dr")
        kw.update(zip(names[2:] if len(args) == 1 else names, args))
        if len(args) not in (0, 1, 6):
            raise TypeError("__init__(): incompatible function arguments")
        c = kw.get("compress_dr_max_lum", 0.2)
        kw["compress_dr_max_lum"] = (0.2 if c else 0.0) if isinstance(c, bool) else float(c)
        defaults = dict(lo_percentile=0.0, hi_percentile=0.2, update_every=1, damping=0.3, color_correct=True)
        for k, v in defaults.items():
            kw.setdefault(k, v)
        super().__init__(**kw)
