"""Host-side Python mirror of the reference's hot-path API over the C ABI.

Reference interfaces mirrored (python binding python/src/cpp/client/processing.cpp):
  XYZLut / XYZLutFloat .__call__(range|frame)   :340-357, 640-700
  destagger(info|shifts, field, inverse)         :527-638
Arrays may be numpy arrays (host) or torch tensors (host or CUDA); CUDA tensors are used
in place (zero copy), host arrays are staged by the C library.  A call given no `stream=` runs on
the torch current stream when its data are CUDA tensors, else on the library's stream (_stream_for).
"""
import ctypes as C

import math

import numpy as np

from . import _capi
from ._capi import CloudIO, check, lib


def device_count():
    return lib.ob_device_count()


def kernel_launch_count(name=None):
    """Kernels launched since load; `name` restricts the count to one family.

    Families: "decode" (K2, any kernel) with its sub-family "decode_pipe" (pipelined K2), "cloud" (K1),
    "normals", "voxel", "voxel_map", "icp", "align", "zone", "image", "frame_ops", "pose", "dewarp",
    "destagger", "lut" and "encode" (K4).  Every launch is in exactly one family, so the total is the sum of
    the families other than "decode_pipe".  Kernels CUB launches inside sorts and scans are not counted.
    """
    if name is not None:
        return lib.ob_kernel_launch_count_of(name.encode())
    return lib.ob_kernel_launch_count()


def set_tunable(name, value, device=0):
    check(lib.ob_set_tunable(device, name.encode(), int(value)))


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _ptr(x):
    if x is None:
        return None
    if _is_torch(x):
        assert x.is_contiguous(), "tensors must be contiguous"
        return x.data_ptr()
    assert x.flags["C_CONTIGUOUS"], "arrays must be C-contiguous"
    return x.ctypes.data


def _itemsize(x):
    return x.element_size() if _is_torch(x) else x.dtype.itemsize


def _np_dtype(x):
    if _is_torch(x):
        import torch
        return {torch.float32: np.dtype(np.float32), torch.float64: np.dtype(np.float64),
                torch.uint8: np.dtype(np.uint8), torch.int32: np.dtype(np.int32),
                torch.uint32: np.dtype(np.uint32), torch.int64: np.dtype(np.int64),
                torch.uint16: np.dtype(np.uint16), torch.int16: np.dtype(np.int16),
                torch.uint64: np.dtype(np.uint64), torch.int8: np.dtype(np.int8)}[x.dtype]
    return x.dtype


def _contig(a, dtype=None, floats=False):
    """`a` (numpy array or torch tensor) made contiguous in its own memory.  dtype: a numpy dtype to convert to; a
    torch tensor is converted only to a floating dtype, since device data carries unsigned integers in signed
    tensors of the same width.  floats: float32 and float64 stay, anything else becomes float64."""
    if _is_torch(a):
        import torch
        if floats and a.dtype not in (torch.float32, torch.float64):
            a = a.double()
        elif dtype is not None and np.dtype(dtype).kind == "f":
            a = a.to(getattr(torch, np.dtype(dtype).name))
        return a.contiguous()
    a = np.ascontiguousarray(a, dtype)
    return a.astype(np.float64) if floats and a.dtype not in (np.float32, np.float64) else a


def _empty(ref, shape, dtype, fill=None):
    """Output of a call on `ref`: a torch tensor on ref's device when ref is a CUDA tensor, else a numpy array, of
    numpy `dtype` (unsigned integers wider than a byte come as the signed torch type of the same width: same bits),
    filled with `fill` when given."""
    dtype = np.dtype(dtype)
    if _is_torch(ref) and ref.is_cuda:
        import torch
        tdt = getattr(torch, dtype.name[1:] if dtype.kind == "u" and dtype.itemsize > 1 else dtype.name)
        if fill is None:
            return torch.empty(shape, dtype=tdt, device=ref.device)
        return torch.full(shape, fill, dtype=tdt, device=ref.device)
    return np.empty(shape, dtype) if fill is None else np.full(shape, fill, dtype)


class _Handle:
    """Base of the objects that own a C handle: when one is collected, the C function named by `_release` frees the
    handle held in the attribute named by `_handle`.  An object that only borrows its handle sets `_owned = False`."""
    _release, _handle, _owned = None, "_h", True

    def __del__(self):
        h = getattr(self, self._handle, None)
        if h and self._owned and lib is not None:
            try:
                getattr(lib, self._release)(h)
            except Exception:
                pass
            setattr(self, self._handle, None)


class PinnedBuffer(_Handle):
    """numpy view over cudaHostAlloc'd memory (ob_host_alloc)."""
    _release, _handle = "ob_host_free", "ptr"

    def __init__(self, nbytes):
        p = C.c_void_p()
        check(lib.ob_host_alloc(nbytes, C.byref(p)))
        self.ptr, self.nbytes = p.value, nbytes
        self.raw = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p.value))


def pinned_empty(shape, dtype):
    """Pinned host array; keeps its allocation alive through the `.base` chain."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    buf = PinnedBuffer(max(n, 1))
    arr = buf.raw[:n].view(dtype).reshape(shape)
    arr_holder = _Holder(arr, buf)
    return arr_holder.arr


class _Holder:
    _keep = []

    def __init__(self, arr, buf):
        self.arr = arr
        _Holder._keep.append(buf)  # pinned buffers live for the process (few, large)


class Stream(_Handle):
    """ob_stream: CUDA stream + staging; one per caller thread / sensor stream."""
    _release, _handle = "ob_stream_destroy", "h"

    def __init__(self, device=0, cuda_stream=None):
        h = C.c_void_p()
        if cuda_stream is None:
            check(lib.ob_stream_create(device, C.byref(h)))
        else:
            check(lib.ob_stream_wrap(device, C.c_void_p(cuda_stream), C.byref(h)))
        self.h, self.device = h, device

    @property
    def cuda_stream(self):
        return lib.ob_stream_cuda_handle(self.h)

    def sync(self):
        check(lib.ob_stream_sync(self.h))


_default_streams = {}
_torch_streams = {}


def _stream(stream, device=0):
    if stream is not None:
        return stream
    if device not in _default_streams:
        _default_streams[device] = Stream(device)
    return _default_streams[device]


def _stream_for(x=None, stream=None, device=0):
    """The stream a call on `x` runs on: `stream` when given; for a CUDA tensor, the torch current stream of its
    device, so the call is ordered after the torch work that wrote `x`; otherwise the library's stream of `device`.
    A torch stream is wrapped once per (device, stream) and the wrapper kept: wrapping configures the device's
    memory pool, which a CUDA graph capture must not see, so a captured call reuses the wrapper an earlier call on
    that stream made."""
    if stream is None and _is_torch(x) and x.is_cuda:
        import torch
        key = (x.device.index, torch.cuda.current_stream(x.device).cuda_stream)
        if key not in _torch_streams:
            _torch_streams[key] = Stream(*key)
        return _torch_streams[key]
    return _stream(stream, device)


class XYZLutT(_Handle):
    """XYZLutT<T> (ouster_core/include/ouster/core/xyzlut.h:76-158) with device-resident tables.

    `direction`/`offset` are fetched lazily from the device (the reference keeps host copies)."""
    _release = "ob_lut_destroy"

    def __init__(self, handle, h, w, dtype, device):
        self._h, self.h, self.w, self.dtype, self.device = handle, h, w, np.dtype(dtype), device
        self._host = None

    # -- constructors ----------------------------------------------------------------------
    @classmethod
    def from_arrays(cls, direction, offset, h, w, device=0):
        """XYZLutT(direction, offset, h, w)  (xyzlut.h:135)."""
        dt = _np_dtype(direction)
        if dt not in (np.dtype(np.float32), np.dtype(np.float64)) or _np_dtype(offset) != dt:
            raise ValueError("direction/offset must both be float32 or float64")
        n = h * w * 3
        dn = direction.numel() if _is_torch(direction) else direction.size
        on = offset.numel() if _is_torch(offset) else offset.size
        if dn != n or on != n:
            raise ValueError("unexpected image dimensions")
        hd = C.c_void_p()
        check(lib.ob_lut_create(_capi.OB_F64 if dt == np.float64 else _capi.OB_F32, _ptr(direction),
                                _ptr(offset), h, w, device, C.byref(hd)))
        return cls(hd, h, w, dt, device)

    @classmethod
    def from_intrinsics(cls, w, h, range_unit, beam_to_lidar_transform, transform,
                        azimuth_angles_deg, altitude_angles_deg, dtype=np.float64, device=0):
        """impl::make_xyz_lut(w, h, range_unit, ...)  (ouster_core/src/xyzlut.cpp:11-89)."""
        b2l = np.ascontiguousarray(beam_to_lidar_transform, np.float64).reshape(16)
        tr = np.ascontiguousarray(transform, np.float64).reshape(16)
        az = np.ascontiguousarray(azimuth_angles_deg, np.float64)
        alt = np.ascontiguousarray(altitude_angles_deg, np.float64)
        dt = np.dtype(dtype)
        hd = C.c_void_p()
        check(lib.ob_lut_from_intrinsics(_capi.OB_F64 if dt == np.float64 else _capi.OB_F32, w, h,
                                         range_unit, b2l.ctypes.data, tr.ctypes.data,
                                         az.ctypes.data, az.size, alt.ctypes.data, alt.size,
                                         device, C.byref(hd)))
        return cls(hd, h, w, dt, device)

    @classmethod
    def from_sensor_info(cls, info, use_extrinsics=True, dtype=np.float64, device=0):
        """XYZLutT(const SensorInfo&, bool use_extrinsics) (xyzlut.h:111-112, xyzlut.cpp:91-106).
        `info`: mapping/obj with w, h, beam_to_lidar_transform, lidar_to_sensor_transform,
        sensor_to_body (optional), beam_azimuth_angles, beam_altitude_angles."""
        g = (lambda k, d=None: info.get(k, d)) if isinstance(info, dict) else \
            (lambda k, d=None: getattr(info, k, d))
        RANGE_UNIT = 0.001  # types.h:46
        tr = np.array(g("lidar_to_sensor_transform"), np.float64).reshape(4, 4)
        ext = g("sensor_to_body")
        if use_extrinsics and ext is not None:
            ext = np.array(ext, np.float64).reshape(4, 4).copy()
            ext[:3, 3] /= RANGE_UNIT
            tr = ext @ tr
        return cls.from_intrinsics(g("w"), g("h"), RANGE_UNIT, g("beam_to_lidar_transform"), tr,
                                   g("beam_azimuth_angles"), g("beam_altitude_angles"), dtype, device)

    # -- members ---------------------------------------------------------------------------
    def _download(self):
        if self._host is None:
            d = np.empty((self.h * self.w, 3), self.dtype)
            o = np.empty((self.h * self.w, 3), self.dtype)
            check(lib.ob_lut_download(self._h, d.ctypes.data, o.ctypes.data))
            self._host = (d, o)
        return self._host

    @property
    def direction(self):
        return self._download()[0]

    @property
    def offset(self):
        return self._download()[1]

    def set_analytic(self, enable=True):
        """Opt into the LUT-free projection (ob_lut_set_analytic): direction/offset recomputed in the
        kernels from per-row / per-column tables; <= 1e-5 norm-wise vs the LUT path, not bit-exact.
        Only LUTs built from per-beam intrinsics have the tables (ValueError otherwise)."""
        check(lib.ob_lut_set_analytic(self._h, int(bool(enable))))
        return self

    @property
    def analytic(self):
        return bool(lib.ob_lut_is_analytic(self._h))

    def __call__(self, rng, out=None, stream=None):
        """lut(range) -> (h*w, 3) points, staggered order (xyzlut.h:139-150)."""
        return cartesian(self, rng, out=out, stream=stream)


def XYZLut(info, use_extrinsics=True, device=0):
    """Python `XYZLut` (double), python/src/cpp/client/processing.cpp:640-700."""
    return XYZLutT.from_sensor_info(info, use_extrinsics, np.float64, device)


def XYZLutFloat(info, use_extrinsics=True, device=0):
    """Python `XYZLutFloat`."""
    return XYZLutT.from_sensor_info(info, use_extrinsics, np.float32, device)


def _numel(x):
    return x.numel() if _is_torch(x) else x.size


def cartesian(lut, rng, out=None, stream=None):
    """cartesian(range, lut) / lut(range).  Raises ValueError("unexpected image dimensions")
    on size mismatch (ouster_core/src/xyzlut.cpp:117-119)."""
    if _np_dtype(rng) != np.dtype(np.uint32):
        if _is_torch(rng):
            raise ValueError("range must be uint32")
        rng = np.ascontiguousarray(rng, np.uint32)
    n = _numel(rng)
    own = out is None
    if own:
        out = _empty(rng, (n, 3), lut.dtype)
    st = _stream_for(rng, stream, lut.device)
    check(lib.ob_cartesian(lut._h, _ptr(rng), n, _ptr(out), st.h))
    if own and not (_is_torch(out) and out.is_cuda):
        st.sync()
    return out


def destagger(img, pixel_shift_by_row, inverse=False, out=None, stream=None, device=0):
    """destagger<T>(img, pixel_shift_by_row, inverse) for (H,W) or (H,W,...) images
    (ouster_core/include/ouster/core/impl/lidar_frame_impl.h:733-860)."""
    shape = tuple(img.shape)
    if len(shape) < 2:
        raise ValueError("image must be at least 2-dimensional")
    h, w = shape[0], shape[1]
    k = int(np.prod(shape[2:])) if len(shape) > 2 else 1
    sh = np.ascontiguousarray(pixel_shift_by_row, np.int32)
    own = out is None
    if own:
        if _is_torch(img):
            import torch
            out = torch.empty_like(img)
        else:
            img = np.ascontiguousarray(img)
            out = np.empty_like(img)
    st = _stream_for(img, stream, device)
    check(lib.ob_destagger(_itemsize(img), k, _ptr(img), sh.ctypes.data, sh.size, h, w,
                           int(bool(inverse)), _ptr(out), st.h))
    if own and not (_is_torch(out) and out.is_cuda):
        st.sync()
    return out


def dewarp(points, poses, out=None, stream=None, device=0):
    """dewarp(points (H, W, 3), poses (W, 4, 4)) -> (H, W, 3): per-column pose application
    (python/src/cpp/client/processing.cpp:132-161; pose_util.h:37-59).  float32 or float64."""
    dt = _np_dtype(points)
    if dt not in (np.dtype(np.float32), np.dtype(np.float64)):
        raise ValueError("points must be float32 or float64")
    if not _is_torch(poses):
        poses = np.ascontiguousarray(poses, dt)
    n_points = _numel(points) // 3
    n_poses = _numel(poses) // 16
    if len(points.shape) == 3 and points.shape[1] != n_poses:
        raise RuntimeError("Number of points per set must match number of poses")
    own = out is None
    if own:
        if _is_torch(points):
            import torch
            out = torch.empty_like(points)
        else:
            points = np.ascontiguousarray(points)
            out = np.empty_like(points)
    st = _stream_for(points, stream, device)
    status = lib.ob_dewarp(_capi.OB_F64 if dt == np.float64 else _capi.OB_F32, _ptr(points), _ptr(poses),
                           n_points, n_poses, _ptr(out), st.h)
    if status == _capi.OB_RUNTIME_ERROR:
        raise RuntimeError(lib.ob_last_error().decode())
    check(status)
    if own and not (_is_torch(out) and out.is_cuda):
        st.sync()
    return out


def dewarp_frame(lut, rng, poses, status, timestamps=None, min_range=0.0, max_range=float("inf"),
                 provenance=False, stream=None, out=None, out_count=None):
    """dewarp(lidar_frame, xyzlut, min_range, max_range) (pose_util.h:456-485): project the range
    image, apply each column's body_to_world pose, keep the points with min_range <= r <= max_range
    (metres) of the columns between the first and last valid one, in column-major order.
    The default max_range=inf is passed as 4294967.295 m, the largest window the C ABI takes; any other window whose
    ceil(min_range * 1e3) or floor(max_range * 1e3) lies outside [0, 4294967295] mm raises ValueError, as does a
    frame of more than 25600 rows.
    Returns points [n, 3] (LUT dtype); with provenance=True also (col_idx u32 [n], timestamps u64 [n]).
    One fused GPU launch: nothing but the surviving points is written.
    Asynchronous device form: `out` = CUDA tensor [capacity, 3] of the LUT dtype and `out_count` = CUDA int64
    tensor [1] (inputs in device memory too): nothing waits for the GPU; returns (out, out_count), the count
    being written in stream order (a count above the capacity means the list was cut there)."""
    from ._capi import DewarpFrameIO
    n_px = lut.h * lut.w
    if _numel(rng) != n_px:
        raise ValueError("unexpected image dimensions")
    if max_range == float("inf"):
        max_range = 4294967.295
    rng, poses, status = _contig(rng, np.uint32), _contig(poses, np.float64), _contig(status, np.uint32)
    if _numel(poses) != lut.w * 16 or _numel(status) != lut.w:
        raise ValueError("poses must be [W, 4, 4] and status [W]")
    io = DewarpFrameIO()
    io.range, io.poses, io.status = _ptr(rng), _ptr(poses), _ptr(status)
    io.min_range, io.max_range = float(min_range), float(max_range)
    if out is not None:
        if out_count is None or provenance:
            raise ValueError("the asynchronous form takes out= and out_count= (device tensors) and no provenance")
        io.points, io.capacity = _ptr(out), _numel(out) // 3
        st = _stream_for(rng, stream, lut.device)
        check(lib.ob_dewarp_frame(lut._h, C.byref(io), C.cast(_ptr(out_count), C.POINTER(C.c_size_t)), st.h))
        return out, out_count
    pts = np.empty((n_px, 3), lut.dtype)
    io.points, io.capacity = pts.ctypes.data, n_px
    ci = ts_out = None
    if provenance:
        if timestamps is None:
            raise ValueError("provenance needs the column timestamps")
        timestamps = _contig(timestamps, np.uint64)
        ci, ts_out = np.empty(n_px, np.uint32), np.empty(n_px, np.uint64)
        io.timestamps, io.col_idx, io.timestamps_out = _ptr(timestamps), ci.ctypes.data, ts_out.ctypes.data
    n = C.c_size_t(0)
    st = _stream_for(rng, stream, lut.device)
    check(lib.ob_dewarp_frame(lut._h, C.byref(io), C.byref(n), st.h))
    if provenance:
        return pts[:n.value], ci[:n.value], ts_out[:n.value]
    return pts[:n.value]


DEFAULT_TARGET_DISTANCE_METER = 0.025                    # ouster/algorithm/normals.h:23
DEFAULT_MIN_ANGLE_INCIDENCE_RAD = 1 * np.pi / 180.0     # ouster/algorithm/normals.h:25


def normals(xyz, rng, *args, sensor_origins_xyz=None, pixel_search_range=1,
            min_angle_of_incidence_rad=DEFAULT_MIN_ANGLE_INCIDENCE_RAD,
            target_distance_m=DEFAULT_TARGET_DISTANCE_METER, vertical_subtent=0.0, return_subtent=False,
            stream=None, device=0):
    """algorithm.normals(xyz, range, sensor_origins_xyz, ...) and the dual-return form
    normals(xyz, range, xyz2, range2, sensor_origins_xyz, ...) (python binding of
    ouster_algorithm/include/ouster/algorithm/normals.h:58-108): destaggered (H, W, 3) points and
    (H, W) ranges in, (H, W, 3) unit normals out (a pair for dual returns).  numpy arrays or torch
    tensors (CUDA tensors stay on the device); float32 / float64.  RuntimeError texts as the reference."""
    from ._capi import NormalsIO
    pos = list(args)
    xyz2 = range2 = None
    # dual-return form: the two leading extra positionals are arrays (xyz2, range2); in the single-return
    # form the second one is the scalar pixel_search_range
    if len(pos) >= 2 and hasattr(pos[0], "shape") and hasattr(pos[1], "shape") and len(pos[1].shape) == 2:
        xyz2, range2 = pos[0], pos[1]
        pos = pos[2:]
    names = ["sensor_origins_xyz", "pixel_search_range", "min_angle_of_incidence_rad", "target_distance_m"]
    kw = {"sensor_origins_xyz": sensor_origins_xyz, "pixel_search_range": pixel_search_range,
          "min_angle_of_incidence_rad": min_angle_of_incidence_rad, "target_distance_m": target_distance_m}
    for nm, v in zip(names, pos):
        kw[nm] = v
    if len(rng.shape) != 2:
        raise RuntimeError("normals: xyz dimensions mismatch")
    h, w = int(rng.shape[0]), int(rng.shape[1])
    dt = _np_dtype(xyz)
    if dt not in (np.dtype(np.float32), np.dtype(np.float64)):
        xyz = np.ascontiguousarray(xyz, np.float64)
        dt = np.dtype(np.float64)
    if _numel(xyz) != h * w * 3:
        raise RuntimeError("normals: xyz dimensions mismatch")
    dual = xyz2 is not None
    if dual:
        if _np_dtype(xyz2) != dt:
            xyz2 = np.ascontiguousarray(xyz2, dt)
        if _numel(xyz2) != h * w * 3:
            raise RuntimeError("normals: xyz dimensions mismatch")
        if tuple(range2.shape) != (h, w):
            raise RuntimeError("normals: range2 dimensions mismatch")
    org = kw["sensor_origins_xyz"]
    if org is None:
        raise TypeError("normals(): incompatible function arguments (sensor_origins_xyz is required)")
    if not _is_torch(org):
        org = np.ascontiguousarray(org, np.float64)
    if len(org.shape) != 2 or org.shape[1] != 3:
        raise TypeError("normals(): incompatible function arguments (sensor_origins_xyz must be (W, 3))")
    if org.shape[0] != w:
        raise RuntimeError("normals: sensor_origins size must match image width")
    xyz, rng = _contig(xyz), _contig(rng, np.uint32)
    on_dev = _is_torch(xyz) and xyz.is_cuda

    def new_out():
        if _is_torch(xyz):
            import torch
            return torch.empty((h, w, 3), dtype=xyz.dtype, device=xyz.device)
        return np.empty((h, w, 3), dt)

    n1 = new_out()
    io = NormalsIO()
    io.n_frames, io.h, io.w = 1, h, w
    io.xyz, io.range, io.normals = _ptr(xyz), _ptr(rng), _ptr(n1)
    n2 = None
    if dual:
        xyz2, range2 = _contig(xyz2), _contig(range2, np.uint32)
        n2 = new_out()
        io.xyz2, io.range2, io.normals2 = _ptr(xyz2), _ptr(range2), _ptr(n2)
    io.sensor_origins_xyz, io.n_origins = _ptr(org), w
    io.pixel_search_range = int(kw["pixel_search_range"])
    io.min_angle_of_incidence_rad = float(kw["min_angle_of_incidence_rad"])
    io.target_distance_m = float(kw["target_distance_m"])
    io.vertical_subtent_rad = float(vertical_subtent)
    sub = np.zeros(1, np.float64)
    io.vertical_subtent_out = sub.ctypes.data
    st = _stream_for(xyz, stream, device)
    status = lib.ob_normals(_capi.OB_F64 if dt == np.float64 else _capi.OB_F32, C.byref(io), st.h)
    if status == _capi.OB_RUNTIME_ERROR:
        raise RuntimeError(lib.ob_last_error().decode())
    check(status)
    if not on_dev or return_subtent:
        st.sync()
    res = (n1, n2) if dual else n1
    return (res, float(sub[0])) if return_subtent else res


VOXEL_MODES = {"first_n": _capi.OB_VOXEL_FIRST_N_POINT, "average": _capi.OB_VOXEL_AVERAGE_POINT,
               "random": _capi.OB_VOXEL_RANDOM, "shuffle_first": _capi.OB_VOXEL_SHUFFLE_FIRST,
               "point_normal": _capi.OB_VOXEL_POINT_NORMAL}


def voxel_downsample(points, voxel_size, mode="shuffle_first", normals=None, max_points_per_voxel=1,
                     min_pts_threshold=1, n=None, stream=None, device=0):
    """Voxel-grid downsampling on the GPU (ob_voxel_downsample), one of VOXEL_MODES:
      "shuffle_first"  core::voxel_downsample(frame, voxel_size) (voxel_hash_map.cpp:262-310), the reference's
                       output order and indices exactly;
      "first_n" / "average" / "random"  core::voxel_downsample_xd with that VoxelDownsampleStrategy (:312-393);
      "point_normal"   algorithm::voxel_downsample_with_normals (voxel_downsample.cpp:21-57), `normals` [n, 3].
    points: [n, cols] float32 / float64 (voxel from columns 0-2), numpy or torch (CUDA tensors stay on the device).
    Returns (points [m, cols] float64, indices [m] uint32 -- int32 on the device), with the normals [m, 3] between
    them for "point_normal".  Voxels come out in the order of their first input row (DESIGN 9).
    n: optional device-resident row count (CUDA integer tensor of one int64, e.g. dewarp_frame's out_count); then
    `points` is a buffer of `capacity` rows, nothing waits for the GPU, and the result is capacity-row buffers plus
    a CUDA int64 [1] count of the valid rows, appended to the tuple.  ValueError texts of the reference."""
    from ._capi import VoxelIO
    m = VOXEL_MODES[mode]
    points = _contig(points, floats=True)
    if len(points.shape) != 2:
        raise ValueError("points must be [n, cols]")
    rows, cols = int(points.shape[0]), int(points.shape[1])
    dt = _np_dtype(points)
    nrm = None
    if m == _capi.OB_VOXEL_POINT_NORMAL:
        if normals is None:
            raise ValueError("point_normal needs normals")
        nrm = _contig(normals, floats=True)
        if _np_dtype(nrm) != dt:
            nrm = _contig(nrm, dt)
        if tuple(nrm.shape) != (rows, 3) or cols != 3:
            raise ValueError("voxel_downsample_with_normals expects Nx3 inputs" if cols != 3 or nrm.shape[-1] != 3
                             else "voxel_downsample_with_normals points/normals size mismatch")
    n_dev = None if n is None else _device_rows(n, points)
    out_cols = 3 if m == _capi.OB_VOXEL_POINT_NORMAL else cols
    out = _empty(points, (rows, out_cols), np.float64)
    out_n = _empty(points, (rows, 3), np.float64) if nrm is not None else None
    idx = _empty(points, (rows,), np.uint32)
    io = VoxelIO()
    io.mode, io.dtype = m, _capi.OB_F64 if dt == np.float64 else _capi.OB_F32
    io.points, io.cols, io.normals = _ptr(points), cols, _ptr(nrm)
    io.voxel_size = float(voxel_size)
    io.max_points_per_voxel, io.min_pts_threshold = int(max_points_per_voxel), int(min_pts_threshold)
    io.points_out, io.normals_out, io.indices_out = _ptr(out), _ptr(out_n), _ptr(idx)
    head = (out, out_n, idx) if nrm is not None else (out, idx)
    if n is not None:
        count = _device_count(points)
        io.n_device, io.capacity, io.n_out = n_dev, rows, count.data_ptr()
        check(lib.ob_voxel_downsample(C.byref(io), _stream_for(points, stream, device).h))
        return head + (count,)
    cnt = C.c_size_t(0)
    io.n, io.n_out = rows, C.addressof(cnt)
    check(lib.ob_voxel_downsample(C.byref(io), _stream_for(points, stream, device).h))
    k = cnt.value
    return tuple(a[:k] for a in head)


DBL_MAX = float(np.finfo(np.float64).max)


def _device_rows(n, data):
    """Address of a device-resident row count n (a CUDA int64 tensor of one element) for the rows in `data`, which
    must then be a CUDA tensor too."""
    import torch
    if not (_is_torch(n) and n.is_cuda and n.dtype == torch.int64 and n.numel() == 1):
        raise ValueError("n must be a CUDA int64 tensor with one element")
    if not (_is_torch(data) and data.is_cuda):
        raise ValueError("a device-side row count needs device inputs")
    return n.data_ptr()


def _device_count(like):
    """A zeroed CUDA int64 [1] on `like`'s device: the count word of a call that returns a device-side count."""
    import torch
    return torch.zeros(1, dtype=torch.int64, device=like.device)


def _point_rows(points, n=None, what="add_points expects an Nx3 array", cols=3):
    """(row argument, kept array): an ob_point_rows (PointRows) for [rows, 3] float32 / float64 points, or with
    cols=None an ob_map_rows (MapRows) for float64 [rows, any cols]; numpy or torch.  n: optional CUDA int64 [1]
    device-resident row count, then `points` holds `capacity` rows."""
    from ._capi import MapRows, PointRows
    points = _contig(points, floats=True) if cols else _contig(points, np.float64)
    if len(points.shape) != 2 or (cols and points.shape[1] != cols):
        raise ValueError(what)
    if cols:
        r = PointRows()
        r.dtype = _capi.OB_F64 if _np_dtype(points) == np.float64 else _capi.OB_F32
        r.points = _ptr(points)
    else:
        r = MapRows()
        r.rows, r.cols = _ptr(points), int(points.shape[1])
    if n is None:
        r.n = int(points.shape[0])
    else:
        r.n_device, r.capacity = _device_rows(n, points), int(points.shape[0])
    return r, points


class VoxelMap(_Handle):
    """Device-resident VoxelHashMap3d (ob_voxel_map, voxel_hash_map.cpp:14-247) with first_n_point insertion, or
    VoxelHashMapXd with num_attributes > 0: rows of cols = 3 + num_attributes float64, x, y, z first (DESIGN f-11).
    Points may be numpy arrays or torch tensors (CUDA tensors stay on the device); results are float64 rows of
    `cols` columns.  point_cloud() and the extracted rows list voxels in creation order (DESIGN 9)."""
    _release = "ob_voxel_map_destroy"

    def __init__(self, voxel_size, max_distance=100.0, max_points_per_voxel=20, min_pts_threshold=1, device=0,
                 num_attributes=0):
        h = C.c_void_p()
        check(lib.ob_voxel_map_create_xd(float(voxel_size), float(max_distance), int(max_points_per_voxel),
                                         int(min_pts_threshold), int(num_attributes), device, C.byref(h)))
        self._h, self.device = h, device
        self.voxel_size, self.max_distance = float(voxel_size), float(max_distance)
        self.max_points_per_voxel, self.min_pts_threshold = int(max_points_per_voxel), int(min_pts_threshold)
        self.num_attributes = int(num_attributes)
        self.cols = 3 + self.num_attributes

    def _origin(self, point):
        """The first three values of a point (the 3-d map takes exactly three)."""
        if self.num_attributes == 0:
            return _contig(point, np.float64).reshape(3)
        p = _contig(point, np.float64).reshape(-1)
        if p.shape[0] < 3:
            raise ValueError("VoxelHashMap method expects a (3+attributes)-element point")
        return p[:3].contiguous() if _is_torch(p) else np.ascontiguousarray(p[:3])

    def clear(self, stream=None):
        check(lib.ob_voxel_map_clear(self._h, _stream(stream, self.device).h))

    def size(self, stream=None):
        """(live voxels, stored points); waits for the stream."""
        v, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.ob_voxel_map_size(self._h, C.byref(v), C.byref(p), _stream(stream, self.device).h))
        return v.value, p.value

    def add_points(self, points, n=None, stream=None):
        """Rows of x, y, z (float32 or float64) for the 3-d map; float64 rows of `cols` columns with attributes
        (ob_voxel_map_add_rows).  n: optional CUDA int64 [1] device-resident row count."""
        if self.num_attributes == 0:
            r, keep = _point_rows(points, n)
            check(lib.ob_voxel_map_add_points(self._h, C.byref(r), _stream_for(keep, stream, self.device).h))
            return
        self.add_rows(points, n, stream)

    def add_rows(self, rows, n=None, stream=None):
        """VoxelHashMap::add_points(ArrayXXdR): float64 [rows, cols]; raises ValueError("VoxelHashMap::add_points
        received unexpected point dimension") for another width."""
        r, keep = _point_rows(rows, n, "add_points expects at least Nx(3+num_attributes) columns", cols=None)
        check(lib.ob_voxel_map_add_rows(self._h, C.byref(r), _stream_for(keep, stream, self.device).h))

    def remove_far(self, origin, extract=False, stream=None):
        """remove_voxels_far_from_location(origin); extract=True returns the erased points (numpy [m, cols])."""
        from ._capi import VoxelMapCullIO
        org = self._origin(origin)
        st = _stream_for(org, stream, self.device)
        io = VoxelMapCullIO()
        io.origin = _ptr(org)
        if not extract:
            check(lib.ob_voxel_map_remove_far(self._h, C.byref(io), st.h))
            return None
        cap = self.size(stream=st)[1]
        out = np.empty((cap, self.cols), np.float64)
        cnt = C.c_size_t(0)
        io.extracted, io.capacity, io.n_extracted = _ptr(out), cap, C.addressof(cnt)
        check(lib.ob_voxel_map_remove_far(self._h, C.byref(io), st.h))
        return out[:cnt.value]

    def point_cloud(self, device=False, stream=None):
        """pointcloud(): [m, cols] float64 numpy array, or a CUDA tensor with device=True."""
        st = _stream(stream, self.device)
        cap = self.size(stream=st)[1]
        cnt = C.c_size_t(0)
        if device:
            import torch
            out = torch.empty((cap, self.cols), dtype=torch.float64, device=torch.device("cuda", self.device))
        else:
            out = np.empty((cap, self.cols), np.float64)
        check(lib.ob_voxel_map_point_cloud(self._h, _ptr(out), cap, C.addressof(cnt), st.h))
        if device:
            st.sync()
        return out[:cnt.value]

    def closest_neighbors(self, points, max_distance_sq=DBL_MAX, n=None, stream=None):
        """get_closest_neighbor for every row of x, y, z: (neighbors [rows, cols], squared distances [rows]) float64,
        torch on the device for CUDA inputs (asynchronous), numpy otherwise."""
        from ._capi import VoxelQueryIO
        r, keep = _point_rows(points, n, "VoxelHashMap method expects a 3-element point")
        rows = int(keep.shape[0])
        nb, d2 = _empty(keep, (rows, self.cols), np.float64, fill=0), _empty(keep, (rows,), np.float64)
        io = VoxelQueryIO()
        io.queries, io.max_distance_sq, io.neighbors, io.distances_sq = r, float(max_distance_sq), _ptr(nb), _ptr(d2)
        st = _stream_for(keep, stream, self.device)
        check(lib.ob_voxel_map_closest_neighbors(self._h, C.byref(io), st.h))
        if not _is_torch(nb):
            st.sync()
        return nb, d2


def icp_align(voxel_map, source, max_distance, kernel_scale, max_num_iterations=50, convergence_criterion=1e-4,
              n=None, stream=None):
    """ICPRegistration::align_points_to_map on the GPU (ob_icp_align): (pose [4, 4] float64, iterations run).
    A CUDA-tensor source gives CUDA tensors (pose float64 [4, 4], iterations int32 [1]) and nothing waits for the
    GPU; n: optional device-resident source row count (e.g. voxel_downsample's count)."""
    from ._capi import IcpIO
    r, keep = _point_rows(source, n)
    io = IcpIO()
    io.source, io.max_distance, io.kernel_scale = r, float(max_distance), float(kernel_scale)
    io.max_num_iterations, io.convergence_criterion = int(max_num_iterations), float(convergence_criterion)
    pose, it = _empty(keep, (4, 4), np.float64), _empty(keep, (1,), np.int32)
    io.pose, io.iterations = _ptr(pose), _ptr(it)
    check(lib.ob_icp_align(voxel_map._h, C.byref(io), _stream_for(keep, stream, voxel_map.device).h))
    return (pose, it) if _is_torch(it) else (pose, int(it[0]))


_FIELD_TAGS = {"uint8": 1, "uint16": 2, "uint32": 3, "uint64": 4, "int8": 5, "int16": 6, "int32": 7, "int64": 8,
               "float32": 9, "float64": 10, "float16": 12}   # ChanFieldType (chanfield.h)
_TAG_BYTES = {1: 1, 2: 2, 3: 4, 4: 8, 5: 1, 6: 2, 7: 4, 8: 8, 9: 4, 10: 8, 12: 2}


def _field_tag(f, dtype):
    """ChanFieldType tag of a map-rows field: the stated type (a numpy dtype or its name, or a tag) when given, else
    the array's own.  A torch int16 / int32 / int64 tensor must state its type: device scans keep uint16 / uint32 /
    uint64 fields in signed tensors of the same width (DeviceLidarScan), so such a tensor does not say which it is.
    A stated type reinterprets the bits and must have the array's element width."""
    if dtype is None:
        name = str(f.dtype).replace("torch.", "")
        if _is_torch(f) and name in ("int16", "int32", "int64"):
            raise ValueError(f"a device {name} field must state its type as (tensor, dtype): unsigned fields of a "
                             "device scan are kept in signed tensors of the same width")
    elif isinstance(dtype, (int, np.integer)) and not isinstance(dtype, bool):
        if int(dtype) not in _TAG_BYTES:
            raise ValueError(f"unsupported field type tag {int(dtype)}")
        tag = int(dtype)
        if _itemsize(f) != _TAG_BYTES[tag]:
            raise ValueError("a field's stated type must have the width of its elements")
        return tag
    else:
        name = np.dtype(dtype).name
    if name not in _FIELD_TAGS:
        raise ValueError(f"unsupported field dtype {name}")
    if _itemsize(f) != _TAG_BYTES[_FIELD_TAGS[name]]:
        raise ValueError("a field's stated type must have the width of its elements")
    return _FIELD_TAGS[name]


def map_rows(items, capacity=None, device_count=None, stream=None):
    """The map exporter's per-return step (map_export.py:589-617) for a list of items, in ONE launch
    (ob_frames_to_map_rows): rows [x, y, z | field channels] float64 for every pixel with range > 0, row-major, item
    i's rows after item i-1's.  An item is None (skipped) or a dict {lut (float64 XYZLutT or pyapi.XYZLut), range
    [h, w] staggered, poses [w, 4, 4] body_to_world, fields: list of [h, w] or [h, w, k] arrays of any integer or float
    type, each either the array or (array, dtype) with its ChanFieldType stated -- required for torch int16 / int32 /
    int64 tensors, which may hold unsigned fields, e.g. (scan.field("SIGNAL"), scan.field_dtype("SIGNAL")) of a
    DeviceLidarScan}; every item must give the same number of columns, and at least one item must be present.
    capacity: rows of the output (default: every pixel).
    device_count (default: True for CUDA-tensor ranges): return (rows [capacity, cols] CUDA tensor, count CUDA int64
    [1]) and let nothing wait -- the count feeds VoxelMap.add_points(n=...); a count above capacity means the list
    was cut there.  Otherwise the rows [n, cols] (numpy for host inputs)."""
    from ._capi import MapField, MapRowsItem
    live = [it for it in items if it is not None]
    if not live:
        raise ValueError("map_rows needs at least one item")
    ref = _contig(live[0]["range"], np.uint32)
    on_dev = _is_torch(ref) and ref.is_cuda
    if device_count is None:
        device_count = on_dev
    if device_count and not on_dev:
        raise ValueError("a device-side count needs device inputs")
    ios = (MapRowsItem * len(live))()
    keep, tables, cols, npx = [], [], None, 0
    for i, it in enumerate(live):
        lut = getattr(it["lut"], "_lut", it["lut"])
        rng, poses = _contig(it["range"], np.uint32), _contig(it["poses"], np.float64)
        if _numel(rng) != lut.h * lut.w:
            raise ValueError("unexpected image dimensions")
        if _numel(poses) != lut.w * 16:
            raise ValueError("poses must be [W, 4, 4]")
        fields = it.get("fields", [])
        tab = (MapField * max(len(fields), 1))()
        c = 3
        for k, f in enumerate(fields):
            f, dtype = f if isinstance(f, tuple) else (f, None)
            f = _contig(f)
            if len(f.shape) not in (2, 3) or tuple(f.shape[:2]) != (lut.h, lut.w):
                raise ValueError("a field must be [h, w] or [h, w, k]")
            ch = 1 if len(f.shape) == 2 else int(f.shape[2])
            tab[k].data, tab[k].type, tab[k].channels = _ptr(f), _field_tag(f, dtype), ch
            c += ch
            keep.append(f)
        if cols is None:
            cols = c
        keep += [rng, poses]
        tables.append(tab)
        ios[i].lut, ios[i].range, ios[i].poses = lut._h, _ptr(rng), _ptr(poses)
        ios[i].fields, ios[i].n_fields = tab, len(fields)
        npx += lut.h * lut.w
    cap = npx if capacity is None else int(capacity)
    out = _empty(ref, (cap, cols), np.float64)
    st = _stream_for(ref, stream, getattr(live[0]["lut"], "_lut", live[0]["lut"]).device)
    if device_count:
        n = _device_count(ref)
        check(lib.ob_frames_to_map_rows(ios, len(live), _ptr(out), cols, cap, n.data_ptr(), st.h))
        return out, n
    cnt = C.c_size_t(0)
    check(lib.ob_frames_to_map_rows(ios, len(live), _ptr(out), cols, cap, C.addressof(cnt), st.h))
    return out[:cnt.value]


def _align_arrays(points, normals, n, what):
    """(PointRows, kept points, kept normals or None) with the normals converted to the points' dtype and memory."""
    r, keep = _point_rows(points, n, f"{what} expects an Nx3 array")
    if normals is None:
        return r, keep, None
    if _is_torch(keep):
        import torch
        normals = torch.as_tensor(normals, device=keep.device)
    elif _is_torch(normals):
        normals = normals.cpu().numpy()
    nk = _contig(normals, _np_dtype(keep))
    if len(nk.shape) != 2 or nk.shape[1] != 3:
        raise ValueError(f"{what} normals must be Nx3")
    return r, keep, nk


def cloud_align(source, target, source_normals=None, target_normals=None, initial_guess=None, max_corr_dist=0.25,
                max_normal_angle_deg=20.0, n_source=None, n_target=None, stream=None):
    """point_to_point_align (no normals) or point_to_plane_align (both normals) on the GPU (ob_cloud_align):
    (pose [4, 4] float64, iterations that reached the solve).  CUDA-tensor clouds give CUDA tensors (pose float64
    [4, 4], iterations int32 [1]) and nothing waits for the GPU; n_source / n_target: optional device-resident row
    counts (e.g. voxel_downsample's count), the arrays then holding `capacity` rows.  initial_guess may be a
    CUDA tensor."""
    from ._capi import CloudAlignIO
    plane = source_normals is not None or target_normals is not None
    if plane and (source_normals is None or target_normals is None):
        raise ValueError("point-to-plane alignment needs both source_normals and target_normals")
    sr, s, sn = _align_arrays(source, source_normals, n_source, "source_points")
    tr, t, tn = _align_arrays(target, target_normals, n_target, "target_points")
    if _is_torch(s) != _is_torch(t) or (_is_torch(s) and s.device != t.device):
        raise ValueError("source and target must live in the same memory")
    if s.dtype != t.dtype:  # the C ABI takes one dtype for both clouds
        s, t, sn, tn = (None if a is None else _contig(a, np.float64) for a in (s, t, sn, tn))
        sr.dtype = tr.dtype = _capi.OB_F64
        sr.points, tr.points = _ptr(s), _ptr(t)
    # ob_cloud_align checks these too; here they also hold on a machine without a GPU (no stream to create yet)
    if not math.isfinite(float(max_corr_dist)) or float(max_corr_dist) <= 0.0:
        raise ValueError("max_corr_dist must be finite and greater than zero")
    if plane:
        a = float(max_normal_angle_deg)
        if not math.isfinite(a) or a < 0.0 or a > 180.0:
            raise ValueError("max_normal_angle_deg must be finite and in [0, 180]")
        if int(sn.shape[0]) != int(s.shape[0]):
            raise ValueError("source_points and source_normals must have the same number of rows")
        if int(tn.shape[0]) != int(t.shape[0]):
            raise ValueError("target_points and target_normals must have the same number of rows")
    io = CloudAlignIO()
    io.mode = _capi.OB_ALIGN_POINT_TO_PLANE if plane else _capi.OB_ALIGN_POINT_TO_POINT
    io.source, io.target = sr, tr
    if plane:
        io.source_normals, io.source_normal_rows = _ptr(sn), int(sn.shape[0])
        io.target_normals, io.target_normal_rows = _ptr(tn), int(tn.shape[0])
    g = None
    if initial_guess is not None:
        g = _contig(initial_guess, np.float64)
        if _numel(g) != 16:
            raise ValueError("initial_guess must be 4x4")
        io.initial_guess = _ptr(g)
    io.max_corr_dist, io.max_normal_angle_deg = float(max_corr_dist), float(max_normal_angle_deg)
    pose, it = _empty(s, (4, 4), np.float64), _empty(s, (1,), np.int32)
    io.pose, io.iterations = _ptr(pose), _ptr(it)
    check(lib.ob_cloud_align(C.byref(io), _stream_for(s, stream).h))
    return (pose, it) if _is_torch(it) else (pose, int(it[0]))


def cloud_nearest(target, queries, cell_size, max_dist_sq, target_normals=None, n_target=None, n_queries=None,
                  stream=None):
    """SpatialHashGrid3D(target[, target_normals], cell_size).nearest(target, q, max_dist_sq) for every query row
    (ob_cloud_nearest): int32 row indices into target, -1 for none.  A CUDA-tensor target and queries give a CUDA
    tensor and nothing waits for the GPU; numpy in, numpy out."""
    from ._capi import CloudNearestIO
    tr, t, tn = _align_arrays(target, target_normals, n_target, "target_points")
    qr, q = _point_rows(queries, n_queries, "queries expects an Nx3 array")
    if _is_torch(t) != _is_torch(q) or (_is_torch(t) and t.device != q.device):
        raise ValueError("target and queries must live in the same memory")
    if t.dtype != q.dtype:
        t, q, tn = (None if a is None else _contig(a, np.float64) for a in (t, q, tn))
        tr.dtype = qr.dtype = _capi.OB_F64
        tr.points, qr.points = _ptr(t), _ptr(q)
    io = CloudNearestIO()
    io.target, io.queries = tr, qr
    io.target_normals = None if tn is None else _ptr(tn)
    io.cell_size, io.max_dist_sq = float(cell_size), float(max_dist_sq)
    out = _empty(q, (int(q.shape[0]),), np.int32, fill=-1)
    io.indices = _ptr(out)
    check(lib.ob_cloud_nearest(C.byref(io), _stream_for(q, stream).h))
    return out


def _align_clouds_input(a, ref=None):
    """(array kept for the call, its columns): numpy or torch rows of float32 / float64; with `ref`, in ref's dtype
    and memory."""
    if ref is not None:
        if _is_torch(ref):
            import torch
            a = torch.as_tensor(a, device=ref.device)
        elif _is_torch(a):
            a = a.cpu().numpy()
        a = _contig(a, _np_dtype(ref))
    else:
        a = _contig(a, floats=True)
    cols = int(a.shape[1]) if len(a.shape) == 2 else 0
    return a, cols


def align_clouds(source, target, source_normals=None, target_normals=None, initial_guess=None,
                 compute_confidence=False, n_source=None, n_target=None, trace=False, stream=None):
    """The point-cloud overloads of algorithm::align_clouds on the GPU (ob_align_clouds): (pose [4, 4] float64,
    confidence), plus a dict of ob_align_clouds_trace (with the target's raw BEV grids and Z histogram) when
    trace=True.  Normals are optional, for both clouds or neither.  CUDA-tensor clouds give a CUDA pose [4, 4] and
    confidence [1] (both float64); n_source / n_target: optional device-resident row counts (e.g. voxel_downsample's
    count), the arrays then holding `capacity` rows.  initial_guess (identity when None) may be a CUDA tensor."""
    from ._capi import AlignCloudsIO, AlignCloudsTrace
    s, s_cols = _align_clouds_input(source)
    if _is_torch(s) != _is_torch(target):
        raise ValueError("source and target must live in the same memory")
    t, t_cols = _align_clouds_input(target, s)
    io = AlignCloudsIO()
    io.source_cols, io.target_cols = s_cols, t_cols
    keep = [s, t]
    for rows, arr, n in ((io.source, s, n_source), (io.target, t, n_target)):
        rows.dtype = _capi.OB_F64 if _np_dtype(arr) == np.float64 else _capi.OB_F32
        rows.points = _ptr(arr)
        if n is None:
            rows.n = int(arr.shape[0]) if len(arr.shape) else 0
        else:
            rows.n_device, rows.capacity = _device_rows(n, arr), int(arr.shape[0])
    if source_normals is not None:
        sn, io.source_normal_cols = _align_clouds_input(source_normals, s)
        io.source_normals, io.source_normal_rows = _ptr(sn), int(sn.shape[0]) if len(sn.shape) else 0
        keep.append(sn)
    if target_normals is not None:
        tn, io.target_normal_cols = _align_clouds_input(target_normals, t)
        io.target_normals, io.target_normal_rows = _ptr(tn), int(tn.shape[0]) if len(tn.shape) else 0
        keep.append(tn)
    g = None
    if initial_guess is not None:
        g = _contig(initial_guess, np.float64)
        if _numel(g) != 16:
            raise ValueError("initial_guess must be 4x4")
        io.initial_guess = _ptr(g)
    io.compute_confidence = int(bool(compute_confidence))
    pose, conf = _empty(s, (4, 4), np.float64), _empty(s, (1,), np.float64)
    io.pose, io.confidence = _ptr(pose), _ptr(conf)
    tr, bufs = None, None
    if trace:
        tr = AlignCloudsTrace()
        bufs = (np.zeros(_capi.OB_ALIGN_MAX_FINE_BASE ** 2), np.zeros(_capi.OB_ALIGN_MAX_COARSE_BASE ** 2),
                np.zeros(_capi.OB_ALIGN_Z_BINS))
        tr.target_fine_grid, tr.target_coarse_grid, tr.target_z_hist = (b.ctypes.data for b in bufs)
        io.trace = C.pointer(tr)
    # ob_align_clouds checks these too, in this order; here they also hold on a machine without a GPU (no stream to
    # create yet)
    for p, nrm, pc, nc, rows in (("source", source_normals, s_cols, io.source_normal_cols, io.source_normal_rows),
                                 ("target", target_normals, t_cols, io.target_normal_cols, io.target_normal_rows)):
        if pc != 3:
            raise ValueError(f"{p}_points must have shape (N, 3)")
        if nrm is not None and nc != 3:
            raise ValueError(f"{p}_normals must have shape (N, 3)")
        pr = io.source if p == "source" else io.target
        if nrm is not None and rows != (pr.capacity if pr.n_device else pr.n):
            raise ValueError(f"{p}_points and {p}_normals must have the same number of rows")
    if (source_normals is None) != (target_normals is None):
        raise ValueError("source_normals and target_normals must both be given or both be omitted")
    check(lib.ob_align_clouds(C.byref(io), _stream_for(s, stream).h))
    out = (pose, conf) if _is_torch(conf) else (pose, float(conf[0]))
    if not trace:
        return out
    d = {name: getattr(tr, name) for name, _ in AlignCloudsTrace._fields_
         if not name.startswith("pad") and not name.endswith(("_grid", "_hist"))}
    for k in ("coarse_scores", "fine_scores", "initial_pose", "icp_poses", "stage_ms"):
        d[k] = np.array(d[k][:], np.float64)
    for k in ("fine_z_bins", "fine_dx", "fine_dy"):
        d[k] = np.array(d[k][:], np.int32)
    d["initial_pose"] = d["initial_pose"].reshape(4, 4)
    d["icp_poses"] = d["icp_poses"].reshape(3, 4, 4)
    fb, cb = tr.fine_base_n, tr.coarse_base_n
    d["target_fine_grid"] = bufs[0][:fb * fb].reshape(fb, fb).copy() if tr.searched else None
    d["target_coarse_grid"] = bufs[1][:cb * cb].reshape(cb, cb).copy() if tr.searched else None
    d["target_z_hist"] = bufs[2].copy() if tr.searched else None
    return out + (d,)


def icp_linear_system(source, target, kernel_scale, stream=None, device=0):
    """build_linear_system(correspondences, kernel_scale) (icp_registration.cpp) on the GPU with the reference's
    deterministic-reduce tree: (jtj [6, 6], lower triangle, jtr [6]) float64 numpy arrays."""
    from ._capi import IcpSystemIO
    s, t = _contig(source, np.float64), _contig(target, np.float64)  # the C ABI reads dense float64 rows
    if tuple(s.shape) != tuple(t.shape) or len(s.shape) != 2 or s.shape[1] != 3:
        raise ValueError("source and target must both be [n, 3]")
    if _is_torch(s) != _is_torch(t) or (_is_torch(s) and s.device != t.device):
        raise ValueError("source and target must live in the same memory")
    jtj, jtr = np.empty((6, 6), np.float64), np.empty(6, np.float64)
    io = IcpSystemIO()
    io.source, io.target, io.n, io.kernel_scale = _ptr(s), _ptr(t), int(s.shape[0]), float(kernel_scale)
    io.jtj, io.jtr = jtj.ctypes.data, jtr.ctypes.data
    check(lib.ob_icp_linear_system(C.byref(io), _stream_for(s, stream, device).h))
    return jtj, jtr


def dewarp_frames(frames, min_range=0.0, max_range=float("inf"), provenance=False, stream=None):
    """dewarp(frame_set, xyzluts, min_range, max_range) (pose_util.h:475, impl/dewarp_impl.h:84-117):
    `frames` is a list with one entry per slot of the set -- None for an empty slot, else a dict
    {lut, range, poses, status[, timestamps]} -- and the result is the concatenation of the frames'
    dewarped points in slot order.  provenance=True also returns (frame_idx, col_idx, timestamps).
    The range window and row limit are dewarp_frame's (the default max_range=inf is passed as 4294967.295 m).
    One launch for the whole set."""
    from ._capi import DewarpFramesIO
    n = len(frames)
    ios = (DewarpFramesIO * max(n, 1))()
    keep, cap, lut0 = [], 0, None
    for i, fr in enumerate(frames):
        if fr is None:
            continue
        lut = fr["lut"]
        lut0 = lut0 or lut
        rng, poses, status = _contig(fr["range"], np.uint32), _contig(fr["poses"], np.float64), \
            _contig(fr["status"], np.uint32)
        if _numel(rng) != lut.h * lut.w:
            raise ValueError("unexpected image dimensions")
        if _numel(poses) != lut.w * 16 or _numel(status) != lut.w:
            raise ValueError("poses must be [W, 4, 4] and status [W]")
        ts = fr.get("timestamps")
        if provenance:
            if ts is None:
                raise ValueError("provenance needs the column timestamps")
            ts = _contig(ts, np.uint64)
        keep += [rng, poses, status, ts]
        ios[i].lut, ios[i].range, ios[i].poses, ios[i].status = lut._h, _ptr(rng), _ptr(poses), _ptr(status)
        ios[i].timestamps = _ptr(ts) if provenance else None
        cap += lut.h * lut.w
    if lut0 is None:
        empty = np.empty((0, 3), np.float64)
        return (empty, np.empty(0, np.uint32), np.empty(0, np.uint32), np.empty(0, np.uint64)) if provenance else empty
    st = _stream(stream, lut0.device)
    if max_range == float("inf"):
        max_range = 4294967.295
    pts = np.empty((cap, 3), lut0.dtype)
    fi = ci = ts_out = None
    if provenance:
        fi, ci, ts_out = np.empty(cap, np.uint32), np.empty(cap, np.uint32), np.empty(cap, np.uint64)
    counts = (C.c_size_t * max(n, 1))()
    total = C.c_size_t(0)
    check(lib.ob_dewarp_frames(ios, n, float(min_range), float(max_range), pts.ctypes.data, cap,
                               fi.ctypes.data if provenance else None, ci.ctypes.data if provenance else None,
                               ts_out.ctypes.data if provenance else None, counts, C.byref(total), st.h))
    k = total.value
    if provenance:
        return pts[:k], fi[:k], ci[:k], ts_out[:k]
    return pts[:k]


def interp_pose(x_interp, x_known, poses_known, two_pose=False, error=None, out=None, stream=None, device=0):
    """ob_interp_pose: x_interp (n,) and x_known (m,) of float64 or int64 (an integer x is read as int64, anything
    else as float64), poses_known (m, 4, 4) of float32 or float64 -> (n, 4, 4) of the poses' dtype, numpy in and
    out, or CUDA tensors on their device.  two_pose: x_known = (t0, t1), the interp_pose(x, t0, x0, t1, x1) form.
    error: a device int64 tensor of 3 words (kind, index, 0) written in stream order; nothing waits, and a failing
    call leaves `out` unwritten.  Without it, errors raise ValueError with the reference's texts."""
    def xconv(a):
        if _is_torch(a):
            import torch
            return a.contiguous() if a.dtype in (torch.int64, torch.float64) else \
                a.to(torch.int64 if not a.is_floating_point() else torch.float64).contiguous()
        a = np.asarray(a)
        return np.ascontiguousarray(a, np.int64 if a.dtype.kind in "iu" else np.float64)
    x, k = xconv(x_interp).reshape(-1), xconv(x_known).reshape(-1)
    if _np_dtype(x) != _np_dtype(k):
        raise ValueError("x_interp and x_known must have one dtype")
    pk = _contig(poses_known, floats=True)
    n, m = _numel(x), _numel(k)
    if _numel(pk) != m * 16:
        raise ValueError("x_known and poses_known sizes are not matching")
    pdt = _np_dtype(pk)
    if out is None:
        out = _empty(x if (_is_torch(x) and x.is_cuda) else pk, (n, 4, 4), pdt)
    io = _capi.InterpPoseIO()
    io.x_interp, io.n, io.x_known, io.m = _ptr(x), n, _ptr(k), m
    io.x_dtype = 1 if _np_dtype(x) == np.int64 else 0
    io.pose_dtype = _capi.OB_F64 if pdt == np.float64 else _capi.OB_F32
    io.two_pose, io.poses_known, io.poses, io.error = int(two_pose), _ptr(pk), _ptr(out), _ptr(error)
    st = _stream_for(x, stream, device)
    check(lib.ob_interp_pose(C.byref(io), st.h))
    return out


def frames_interp_pose(frames, t0, x0, t1=None, x1=None, error=None, stream=None, device=0):
    """ob_frames_interp_pose: ConstantVelocityDeskewMethod::update over a frame set.  `frames`: one entry per slot,
    None for an empty slot, else (timestamps (W,) uint64, status (W,) uint32, poses (W, 4, 4) float64, written in
    place) -- numpy arrays or CUDA tensors, e.g. the column headers core.Decoder.decode writes (uint64 / uint32 data
    in int64 / int32 tensors).  x0 / x1: 4 x 4 float64, host or device; x1 None: every valid column gets x0.
    error: optional device int64 tensor of 3 words (kind, column, slot); nothing waits with device buffers."""
    items = (_capi.FramePosesItem * max(len(frames), 1))()
    keep, ref = [], None
    for i, fr in enumerate(frames):
        if fr is None:
            continue
        ts, stt, poses = fr
        w = _numel(ts)
        if _numel(stt) != w or _numel(poses) != w * 16:
            raise ValueError("timestamps, status and poses must be [W], [W] and [W, 4, 4]")
        if _is_torch(poses):
            assert poses.is_contiguous(), "poses must be contiguous: they are written in place"
        else:
            assert poses.dtype == np.float64 and poses.flags["C_CONTIGUOUS"], "poses must be C-contiguous float64"
        ts, stt = _contig(ts, np.uint64), _contig(stt, np.uint32)
        keep += [ts, stt]
        ref = ref if ref is not None else poses
        items[i].timestamps, items[i].status, items[i].poses, items[i].w = _ptr(ts), _ptr(stt), _ptr(poses), w
    a0 = _contig(x0, np.float64)
    a1 = None if x1 is None else _contig(x1, np.float64)
    st = _stream_for(ref if ref is not None else a0, stream, device)
    check(lib.ob_frames_interp_pose(items, len(frames), float(t0), _ptr(a0), float(t1 if t1 is not None else 0.0),
                                    _ptr(a1), _ptr(error), st.h))


_GROUND_GRIDS = (("valid", np.uint8), ("obstacle", np.uint8), ("floor_z", np.float64), ("height", np.float64),
                 ("roughness", np.float64))


def ground_mask(frames, grid_size=0.5, stop=None, model=False, stream=None):
    """ob_ground_mask: impl::get_ground_mask (ground_seg.cpp:1137-1314) over a frame set, one call for all frames.

    `frames`: one entry per slot, None for an empty slot, else a dict {lut (a float64 XYZLutT built with
    extrinsics), ranges (list of (H, W) uint32, one per return), status (W,), poses (W, 4, 4) float64[, normals,
    normals2 (H, W, 3) float32: the NORMALS / NORMALS2 fields][, sensor_to_body (4, 4): given without normals, the
    call computes the normals get_ground_mask would][, masks: contiguous (H, W) uint8 outputs, one per return]} --
    numpy arrays or CUDA tensors; the masks of a frame
    whose first range image is a CUDA tensor are CUDA tensors.  stop: the pass to stop after (an index into
    _capi.GROUND_STAGES; default the last); masks are classified only after the last pass and are zero otherwise.
    model=True also returns each frame's model after pass `stop`: its header and five (rows, cols) grids, on the
    masks' side (a first call stopped after the cells pass learns the grid shapes).
    -> list with, per slot, None or {"masks": [one (H, W) uint8 per return], and with model=True "model" (dict of
    the ob_ground_model fields), "grids" (dict, None without a grid), "prune_levels"}; a frame whose normals were
    computed also has "vertical_subtent" (the subtent they used).  Errors raise ValueError with
    the reference's texts."""
    stop = _capi.OB_GROUND_FINAL if stop is None else int(stop)
    n = len(frames)
    items = (_capi.GroundItem * max(n, 1))()
    keep, out, ref, dev = [], [None] * n, None, 0
    for i, fr in enumerate(frames):
        if fr is None:
            continue
        lut = fr["lut"]
        h, w = lut.h, lut.w
        rngs = [_contig(r, np.uint32) for r in fr["ranges"]]
        for r in rngs:
            if _numel(r) != h * w:
                raise ValueError("unexpected image dimensions")
        status, poses = _contig(fr["status"], np.uint32), _contig(fr["poses"], np.float64)
        if _numel(status) != w or _numel(poses) != w * 16:
            raise ValueError("poses must be [W, 4, 4] and status [W]")
        nrm = [None if fr.get(k) is None else _contig(fr[k], np.float32) for k in ("normals", "normals2")]
        for x in nrm:
            if x is not None and _numel(x) != h * w * 3:
                raise ValueError("normals must be [H, W, 3]")
        s2b = None
        if nrm[0] is None and fr.get("sensor_to_body") is not None:
            s2b = _contig(fr["sensor_to_body"], np.float64)
        masks = fr.get("masks") or [_empty(rngs[0] if rngs else status, (h, w), np.uint8) for _ in rngs]
        rp = (C.c_void_p * max(len(rngs), 1))(*[_ptr(r) for r in rngs])
        mp = (C.c_void_p * max(len(masks), 1))(*[_ptr(m) for m in masks])
        sub = np.zeros(1)
        keep += [rngs, status, poses, nrm, masks, rp, mp, s2b, sub]
        it = items[i]
        it.lut, it.h, it.w, it.n_returns = lut._h, h, w, len(rngs)
        it.range = C.cast(rp, C.POINTER(C.c_void_p)) if rngs else None
        it.status, it.poses, it.normals, it.normals2 = _ptr(status), _ptr(poses), _ptr(nrm[0]), _ptr(nrm[1])
        it.masks, it.n_masks, it.mask_h, it.mask_w = C.cast(mp, C.POINTER(C.c_void_p)), len(masks), h, w
        out[i] = {"masks": masks}
        if s2b is not None:
            it.sensor_to_body, it.compute_normals, it.vertical_subtent_out = _ptr(s2b), 1, sub.ctypes.data
            out[i]["_sub"] = sub
        if ref is None:
            ref, dev = (rngs[0] if rngs else status), lut.device
    st = _stream_for(ref, stream, dev)
    def done():
        for o in out:
            if o is not None and "_sub" in o:
                o["vertical_subtent"] = float(o.pop("_sub")[0])
        return out
    if not model:
        check(lib.ob_ground_mask(items, n, float(grid_size), stop, st.h))
        return done()
    headers = [_capi.GroundModel() for _ in range(n)]
    levels = np.zeros(n, np.int32)
    for i in range(n):
        if out[i] is not None:
            items[i].model = C.addressof(headers[i])
    check(lib.ob_ground_mask(items, n, float(grid_size), _capi.GROUND_STAGES.index("cells"), st.h))
    for i in range(n):
        if out[i] is None:
            continue
        hd = headers[i]
        cells = int(hd.rows) * int(hd.cols)
        grids = None
        if cells > 0:
            like = out[i]["masks"][0] if out[i]["masks"] else None
            grids = {k: _empty(like, (hd.rows, hd.cols), dt) for k, dt in _GROUND_GRIDS}
            keep.append(grids)
            for k, _ in _GROUND_GRIDS:
                setattr(items[i], k, _ptr(grids[k]))
            items[i].grid_capacity = cells
        items[i].prune_levels = levels.ctypes.data + 4 * i
        out[i]["grids"] = grids
    check(lib.ob_ground_mask(items, n, float(grid_size), stop, st.h))
    st.sync()
    for i in range(n):
        if out[i] is not None:
            out[i]["model"] = {k: getattr(headers[i], k) for k, _ in _capi.GroundModel._fields_}
            out[i]["prune_levels"] = int(levels[i])
    return done()


def transform(points, pose, out=None, stream=None, device=0):
    """transform(points (..., 3), pose (4, 4)): one pose for every point (pose_util.h:118-131)."""
    pose = pose if _is_torch(pose) else np.ascontiguousarray(pose, _np_dtype(points)).reshape(1, 16)
    shape = tuple(points.shape)
    flat = points.reshape(-1, 3)
    res = dewarp(flat, pose, out=None if out is None else out.reshape(-1, 3), stream=stream, device=device)
    return res.reshape(shape)


def plan_scan_to_cloud(lut, pixel_shift_by_row, rng, xyz=None, range_destaggered=None,
                       xyz_destaggered=None, stream=None, poses=None):
    """Marshal an ob_scan_to_cloud call once and return a callable that launches it (`plan()`): for
    steady-state callers that process into the same buffers every step.  Arguments as scan_to_cloud."""
    st = _stream(stream, lut.device)
    F, R, H, W = tuple(rng.shape)
    io = CloudIO()
    io.n_frames, io.n_returns = F, R
    n = H * W
    io.range, io.range_frame_stride, io.range_return_stride = _ptr(rng), R * n, n
    if xyz is not None:
        io.xyz, io.xyz_frame_stride, io.xyz_return_stride = _ptr(xyz), R * n * 3, n * 3
    if range_destaggered is not None:
        io.range_destaggered, io.rd_frame_stride, io.rd_return_stride = _ptr(range_destaggered), R * n, n
    if xyz_destaggered is not None:
        io.xyz_destaggered, io.xd_frame_stride, io.xd_return_stride = _ptr(xyz_destaggered), R * n * 3, n * 3
    if poses is not None:
        if _np_dtype(poses) != lut.dtype:
            raise ValueError("poses must have the dtype of the lut")
        pn = _numel(poses)
        if pn == W * 16:
            io.poses, io.poses_frame_stride = _ptr(poses), 0
        elif pn == F * W * 16:
            io.poses, io.poses_frame_stride = _ptr(poses), W * 16
        else:
            raise ValueError("poses must be [W, 4, 4] or [F, W, 4, 4]")
    sh, nsh = None, 0
    if pixel_shift_by_row is not None:
        sh = np.ascontiguousarray(pixel_shift_by_row, np.int32)
        nsh = sh.size
    lut_h, sh_p, io_ref, st_h, run = lut._h, (sh.ctypes.data if sh is not None else None), C.byref(io), st.h, \
        lib.ob_scan_to_cloud

    def plan():
        check(run(lut_h, sh_p, nsh, io_ref, st_h))
    plan._keep = (lut, sh, io, st, rng, xyz, range_destaggered, xyz_destaggered, poses)
    return plan


def scan_to_cloud(lut, pixel_shift_by_row, rng, xyz=None, range_destaggered=None,
                  xyz_destaggered=None, stream=None, poses=None):
    """Fused batch: rng is [F, R, H, W] uint32; outputs [F, R, H*W, 3] (xyz), [F, R, H, W]
    (range_destaggered), [F, R, H, W, 3] (xyz_destaggered).  `poses` ([W, 4, 4] shared by all
    frames or [F, W, 4, 4], LUT dtype, e.g. LidarScan.body_to_world) fuses dewarp(xyz, poses) into
    the same pass.  Asynchronous on `stream`."""
    plan_scan_to_cloud(lut, pixel_shift_by_row, rng, xyz, range_destaggered, xyz_destaggered, stream, poses)()


class Decoder(_Handle):
    """ob_decoder: device-side PacketFormat decode table.

    layout: dict with packet_header_size, col_header_size, channel_data_size, col_size,
            packet_size, columns_per_packet, pixels_per_column, columns_per_frame and the three
            column-header infos col_timestamp / col_measurement_id / col_status as
            (offset, mask, shift) tuples.
    fields: list of dicts {name, offset, mask, shift, elem_size, range_return, zero_pattern}.
    """
    _release = "ob_decoder_destroy"

    def __init__(self, layout, fields, device=0):
        from ._capi import FieldDesc, PacketLayout
        L = PacketLayout()
        for k in ("packet_header_size", "col_header_size", "channel_data_size", "col_size",
                  "packet_size", "columns_per_packet", "pixels_per_column", "columns_per_frame"):
            setattr(L, k, int(layout[k]))
        for k in ("col_timestamp", "col_measurement_id", "col_status"):
            o, m, sft = layout[k]
            setattr(L, k, FieldDesc(int(o), 8, int(m), int(sft), -1, 0, 0))
        arr = (FieldDesc * max(len(fields), 1))()
        for i, f in enumerate(fields):
            arr[i] = FieldDesc(int(f["offset"]), int(f["elem_size"]), int(f["mask"]), int(f["shift"]),
                               int(f.get("range_return", -1)), int(f.get("zero_pattern", 0)), 0)
        h = C.c_void_p()
        check(lib.ob_decoder_create(C.byref(L), arr, len(fields), device, C.byref(h)))
        self._h, self.device = h, device
        self.layout, self.fields = dict(layout), [dict(f) for f in fields]
        self.h_px, self.w_px = int(layout["pixels_per_column"]), int(layout["columns_per_frame"])

    def decode(self, frames, lut=None, pixel_shift_by_row=None, stream=None):
        """frames: list of dicts {packets, n_slots, packet_stride, col_src (np.int32 [W] or None),
        fields: {name: array}, timestamp, measurement_id, status, xyz: [a0, a1],
        range_destaggered: [a0, a1]}.  Asynchronous on `stream`."""
        from ._capi import DecodeIO
        st = _stream(stream, self.device)
        ios = (DecodeIO * len(frames))()
        keep = []
        for i, fr in enumerate(frames):
            io = ios[i]
            io.packets = _ptr(fr["packets"])
            io.n_slots = int(fr["n_slots"])
            io.packet_stride = int(fr["packet_stride"])
            cs = fr.get("col_src")
            if cs is not None:
                cs = np.ascontiguousarray(cs, np.int32)
                keep.append(cs)
                io.col_src = cs.ctypes.data
            outs = fr.get("fields", {})
            for k, f in enumerate(self.fields):
                a = outs.get(f["name"])
                if a is not None:
                    io.fields[k] = _ptr(a)
            for k in ("timestamp", "measurement_id", "status"):
                if fr.get(k) is not None:
                    setattr(io, k, _ptr(fr[k]))
            for r, a in enumerate(fr.get("xyz", []) or []):
                if a is not None:
                    io.xyz[r] = _ptr(a)
            for r, a in enumerate(fr.get("range_destaggered", []) or []):
                if a is not None:
                    io.range_destaggered[r] = _ptr(a)
            if fr.get("lut") is not None:
                io.lut = fr["lut"]._h
        sh, nsh = None, 0
        if pixel_shift_by_row is not None:
            sh = np.ascontiguousarray(pixel_shift_by_row, np.int32)
            nsh = sh.size
        check(lib.ob_decode_frames(self._h, ios, len(frames), lut._h if lut is not None else None,
                                   sh.ctypes.data if sh is not None else None, nsh, st.h))

    @classmethod
    def from_sensor(cls, info, frame, device=0):
        """Decoder for the fields `frame` (host LidarFrame) shares with the sensor's PacketFormat."""
        L = info.layout
        layout = {k: getattr(L, k) for k in ("packet_header_size", "col_header_size", "channel_data_size",
                                             "col_size", "packet_size", "columns_per_packet",
                                             "pixels_per_column", "columns_per_frame")}
        for k in ("col_timestamp", "col_measurement_id", "col_status"):
            d = getattr(L, k)
            layout[k] = (d.offset, d.mask, d.shift)
        fields = []
        have = set(frame.fields)
        for name, tag, off, mask, shift, nel, vm in info.fields():
            if name not in have:
                continue
            a = frame.field(name)
            es = a.dtype.itemsize * (a.shape[2] if a.ndim == 3 else 1)
            fields.append({"name": name, "offset": off, "mask": mask, "shift": shift, "elem_size": es,
                           "range_return": {"RANGE": 0, "RANGE2": 1}.get(name, -1),
                           "zero_pattern": 0x7e00 if name == "RGB" else 0})
        return cls(layout, fields, device)

    def prepare_batch(self, n_frames, packets, n_slots, packet_stride, packets_frame_stride, fields,
                      lut=None, pixel_shift_by_row=None, xyz=None, range_destaggered=None,
                      timestamp=None, measurement_id=None, status=None, stream=None, frame_luts=None):
        """Build the ob_decode_batch descriptor of a uniformly strided batch ONCE and return a callable
        that launches it (`plan()`): a steady-state caller decodes into the same buffers every step, and
        re-marshalling ~100 pointers through ctypes costs more host time than the launch takes on the GPU.
        Arguments as decode_batch."""
        from ._capi import DecodeBatch
        st = _stream(stream, self.device)
        b = DecodeBatch()
        b.n_frames = n_frames
        b.packets, b.n_slots = _ptr(packets), n_slots
        b.packet_stride, b.packets_frame_stride = packet_stride, packets_frame_stride
        n_px = self.h_px * self.w_px
        for k, f in enumerate(self.fields):
            a = fields.get(f["name"])
            if a is not None:
                b.fields[k] = _ptr(a)
                b.field_frame_stride[k] = n_px * f["elem_size"]
        if timestamp is not None:
            b.timestamp, b.timestamp_frame_stride = _ptr(timestamp), self.w_px * 8
        if measurement_id is not None:
            b.measurement_id, b.measurement_id_frame_stride = _ptr(measurement_id), self.w_px * 2
        if status is not None:
            b.status, b.status_frame_stride = _ptr(status), self.w_px * 4
        any_lut = lut if lut is not None else (frame_luts[0] if frame_luts else None)
        esz = 8 if (any_lut is not None and any_lut.dtype == np.float64) else 4
        keep = [packets, fields, xyz, range_destaggered, timestamp, measurement_id, status, lut, frame_luts]
        if frame_luts:
            arr = (C.c_void_p * n_frames)(*[l._h.value for l in frame_luts])
            keep.append(arr)
            b.frame_luts = C.cast(arr, C.POINTER(C.c_void_p))
        for r, a in enumerate(xyz or []):
            if a is not None:
                b.xyz[r] = _ptr(a)
        b.xyz_frame_stride = n_px * 3 * esz
        for r, a in enumerate(range_destaggered or []):
            if a is not None:
                b.range_destaggered[r] = _ptr(a)
        b.rd_frame_stride = n_px * 4
        sh, nsh = None, 0
        if pixel_shift_by_row is not None:
            sh = np.ascontiguousarray(pixel_shift_by_row, np.int32)
            nsh = sh.size
        keep.append(sh)
        dec_h, b_ref, lut_h = self._h, C.byref(b), (lut._h if lut is not None else None)
        sh_p, st_h, run = (sh.ctypes.data if sh is not None else None), st.h, lib.ob_decode_batch_run

        def plan():
            check(run(dec_h, b_ref, lut_h, sh_p, nsh, st_h))
        plan._keep = (keep, b, st)
        return plan

    def decode_batch(self, n_frames, packets, n_slots, packet_stride, packets_frame_stride, fields,
                     lut=None, pixel_shift_by_row=None, xyz=None, range_destaggered=None,
                     timestamp=None, measurement_id=None, status=None, stream=None, frame_luts=None):
        """Uniformly strided batch of complete frames (ob_decode_batch_run).  `fields` maps a field
        name to an array/tensor shaped [n_frames, H, W(, k)]; xyz / range_destaggered are lists (one
        entry per return) of [n_frames, H*W, 3] / [n_frames, H, W] arrays."""
        self.prepare_batch(n_frames, packets, n_slots, packet_stride, packets_frame_stride, fields, lut,
                           pixel_shift_by_row, xyz, range_destaggered, timestamp, measurement_id, status,
                           stream, frame_luts)()


# ---- zone monitoring (DESIGN f-8) -------------------------------------------------------------------------------
ZONE_STATE_DTYPE = np.dtype([("live", np.uint8), ("id", np.uint8), ("error_flags", np.uint8),
                             ("trigger_type", np.uint8), ("trigger_status", np.uint8), ("triggered_frames", np.uint32),
                             ("count", np.uint32), ("occlusion_count", np.uint32), ("invalid_count", np.uint32),
                             ("max_count", np.uint32), ("min_range", np.uint32), ("max_range", np.uint32),
                             ("mean_range", np.uint32)])  # ZoneState, packed: 37 bytes
assert ZONE_STATE_DTYPE.itemsize == 37


def _lut_pair(lut, npx, what):
    """(direction, offset) pointers of a float64 LUT: an XYZLutT of dtype float64 (device tables) or a pair of
    (h*w, 3) float64 arrays / CUDA tensors."""
    if lut is None:
        return None, None, ()
    if isinstance(lut, XYZLutT):
        if lut.dtype != np.float64 or lut.h * lut.w != npx:
            raise ValueError(f"{what} must be a float64 LUT of the zone images' size")
        d, o = C.c_void_p(), C.c_void_p()
        check(lib.ob_lut_device_ptrs(lut._h, C.byref(d), C.byref(o)))
        return d.value, o.value, (lut,)
    d, o = lut
    keep = []
    for a in (d, o):
        a = _contig(a, np.float64)
        if _numel(a) != npx * 3:
            raise ValueError(f"{what} must hold h*w*3 values")
        keep.append(a)
    return _ptr(keep[0]), _ptr(keep[1]), tuple(keep)


def zone_render(zones, h, w, sensor_lut, body_lut=None, device_out=None, stream=None, device=0):
    """Zone::render of every zone in one launch (ob_zone_render).

    zones: sequence of dicts with `triangles` ([n, 9] or [n, 3, 3] float32: v0, v1, v2), `coordinate_frame`
    (1 BODY, 2 SENSOR) and optional `point_count`, `frame_count`, `mode` (default 1, 1, 1 OCCUPANCY).
    sensor_lut / body_lut: BeamConfig's LUTs without / with sensor_to_body (see _lut_pair).
    -> (near_mm, far_mm [n_zones, h, w] uint32, pixels_with_intersections numpy uint32 [n_zones]).  The images are
    CUDA int32 tensors (same bits) when device_out is True, or by default when a LUT lives on the GPU."""
    from ._capi import ZoneDesc, ZoneRenderIO
    zones = list(zones)
    npx = int(h) * int(w)
    sd, so, keep_s = _lut_pair(sensor_lut, npx, "sensor_lut")
    bd, bo, keep_b = _lut_pair(body_lut, npx, "body_lut")
    descs = (ZoneDesc * max(len(zones), 1))()
    tris = []
    for i, z in enumerate(zones):
        t = np.ascontiguousarray(z["triangles"], np.float32).reshape(-1, 9)
        tris.append(t)
        descs[i].triangles, descs[i].n_triangles = t.ctypes.data, len(t)
        descs[i].coordinate_frame = int(z["coordinate_frame"])
        descs[i].point_count = int(z.get("point_count", 1))
        descs[i].frame_count = int(z.get("frame_count", 1))
        descs[i].mode = int(z.get("mode", _capi.OB_ZONE_MODE_OCCUPANCY))
    on_dev = [a for a in keep_s + keep_b if (isinstance(a, XYZLutT) or (_is_torch(a) and a.is_cuda))]
    if device_out is None:
        device_out = bool(on_dev)
    ref = None  # an empty CUDA tensor on the output device when the images stay there
    if device_out:
        import torch
        dev = on_dev[0].device if on_dev else device
        ref = torch.empty(0, device=torch.device("cuda", dev) if isinstance(dev, int) else dev)
    shape = (len(zones), int(h), int(w))
    near, far = _empty(ref, shape, np.uint32), _empty(ref, shape, np.uint32)
    st = _stream_for(ref, stream, device)
    px = np.zeros(max(len(zones), 1), np.uint32)
    io = ZoneRenderIO()
    io.n_rows, io.n_cols = int(h), int(w)
    io.sensor_direction, io.sensor_offset, io.body_direction, io.body_offset = sd, so, bd, bo
    io.zones, io.n_zones = descs, len(zones)
    io.near_mm, io.far_mm, io.pixels_with_intersections = _ptr(near), _ptr(far), px.ctypes.data
    check(lib.ob_zone_render(C.byref(io), st.h))
    return near, far, px[:len(zones)]


class ZoneMonitor(_Handle):
    """Device-resident EmulatedZoneMon (ob_zone_monitor): up to 16 live zones' near/far images in HBM; update()
    runs _calc_counts and the trigger counters of one frame and leaves the 16 ZoneState records on the device.

    live: sequence of dicts with `id`, `mode`, `point_count`, `frame_count`, `near_mm`, `far_mm` ((h, w) uint32,
    numpy or CUDA) and optional initial `triggers` / `alerts`.  The slot of a zone (its bitmask bit) is its index."""
    _release = "ob_zone_monitor_destroy"

    def __init__(self, live, h, w, device=0):
        from ._capi import ZoneLive
        live = list(live)
        arr = (ZoneLive * max(len(live), 1))()
        keep = []
        for i, z in enumerate(live):
            ims = []
            for k in ("near_mm", "far_mm"):
                a = _contig(z[k], np.uint32)
                if _numel(a) != int(h) * int(w):
                    raise ValueError("zone images must be h x w")
                ims.append(a)
            keep += ims
            arr[i].id, arr[i].mode = int(z["id"]), int(z["mode"])
            arr[i].point_count, arr[i].frame_count = int(z["point_count"]), int(z["frame_count"])
            arr[i].near_mm, arr[i].far_mm = _ptr(ims[0]), _ptr(ims[1])
            arr[i].triggers, arr[i].alerts = int(z.get("triggers", 0)), int(z.get("alerts", 0))
        hd = C.c_void_p()
        check(lib.ob_zone_monitor_create(device, int(h), int(w), arr, len(live), C.byref(hd)))
        self._h, self.h, self.w, self.n_live, self.device = hd, int(h), int(w), len(live), device
        self._st = None

    def update(self, range_img, bitmask=None, stream=None):
        """calc_triggers(range, bitmask): range (h, w) uint32 (numpy, or a CUDA int32 / uint32 tensor such as K2's
        RANGE); bitmask (optional, same shape, uint32 / int32) gets bit `slot` OR-ed where a zone triggers.  CUDA
        inputs: nothing waits for the GPU."""
        if _numel(range_img) != self.h * self.w:
            raise ValueError("range image must be h x w")
        if _is_torch(range_img):
            import torch
            if range_img.dtype not in (torch.int32, torch.uint32):
                raise ValueError("range must be uint32")
        r = _contig(range_img, np.uint32)
        if bitmask is not None:
            # written in place, so neither a copy nor a conversion will do
            if _is_torch(bitmask):
                import torch
                ok = bitmask.dtype in (torch.int32, torch.uint32) and bitmask.is_contiguous()
            else:
                ok = isinstance(bitmask, np.ndarray) and bitmask.dtype in (np.uint32, np.int32) and \
                    bitmask.flags["C_CONTIGUOUS"]
            if not ok or _numel(bitmask) != self.h * self.w:
                raise ValueError("bitmask must be a contiguous h x w uint32 / int32 array")
        st = self._st = _stream_for(r, stream, self.device)
        check(lib.ob_zone_monitor_update(self._h, _ptr(r), None if bitmask is None else _ptr(bitmask), st.h))

    def states(self, device=False, stream=None):
        """The 16 ZoneState records of the last update: numpy (ZONE_STATE_DTYPE) or, with device=True, a CUDA
        uint8 tensor [16, 37] written on the stream without waiting."""
        st = stream or self._st or _stream(None, self.device)
        if device:
            import torch
            out = torch.empty((16, 37), dtype=torch.uint8, device=torch.device("cuda", st.device))
            check(lib.ob_zone_monitor_states(self._h, out.data_ptr(), st.h))
            return out
        out = np.zeros(16, ZONE_STATE_DTYPE)
        check(lib.ob_zone_monitor_states(self._h, out.ctypes.data, st.h))
        return out

    def counters(self, stream=None):
        """(triggers, alerts, range_sums): per-slot lists of the trigger and alert counters and of the exact sum of
        the last update's triggering ranges; waits for the stream."""
        n = max(self.n_live, 1)
        t, a, r = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint64)
        st = stream or self._st or _stream(None, self.device)
        check(lib.ob_zone_monitor_counters(self._h, t.ctypes.data, a.ctypes.data, r.ctypes.data, st.h))
        return ([int(v) for v in t[:self.n_live]], [int(v) for v in a[:self.n_live]],
                [int(v) for v in r[:self.n_live]])


class ImageProcessor(_Handle):
    """Device-resident image post-processor (ob_image_proc): one AutoExposure, BeamUniformityCorrector or
    LocalToneMapper with its state in device memory.  kind: "auto_exposure", "beam_uniformity" or
    "local_tone_map"; the keyword arguments are the constructor's (ignored by beam_uniformity), and those left out
    take the kind's default constructor values."""
    _release = "ob_image_proc_destroy"

    KINDS = {"auto_exposure": _capi.OB_IMAGE_AUTO_EXPOSURE, "beam_uniformity": _capi.OB_IMAGE_BEAM_UNIFORMITY,
             "local_tone_map": _capi.OB_IMAGE_LOCAL_TONE_MAP}
    # the reference's default constructors (image_processing.cpp:201-205, 508-509, header defaults)
    DEFAULTS = {"auto_exposure": dict(lo_percentile=0.1, hi_percentile=0.1, update_every=3, damping=0.9,
                                      compress_dr_max_lum=0.0, color_correct=False),
                "beam_uniformity": dict(lo_percentile=0.0, hi_percentile=0.0, update_every=8, damping=0.92,
                                        compress_dr_max_lum=0.0, color_correct=False),
                "local_tone_map": dict(lo_percentile=0.0, hi_percentile=0.2, update_every=1, damping=0.3,
                                       compress_dr_max_lum=0.2, color_correct=True)}

    def __init__(self, kind, lo_percentile=None, hi_percentile=None, update_every=None, damping=None,
                 compress_dr_max_lum=None, color_correct=None, device=0):
        given = dict(lo_percentile=lo_percentile, hi_percentile=hi_percentile, update_every=update_every,
                     damping=damping, compress_dr_max_lum=compress_dr_max_lum, color_correct=color_correct)
        a = {k: (self.DEFAULTS[kind][k] if v is None else v) for k, v in given.items()}
        p = _capi.ImageParams(float(a["lo_percentile"]), float(a["hi_percentile"]), int(a["update_every"]),
                              int(bool(a["color_correct"])), float(a["damping"]), float(a["compress_dr_max_lum"]))
        hd = C.c_void_p()
        check(lib.ob_image_proc_create(device, self.KINDS[kind], C.byref(p), C.byref(hd)))
        self._h, self.kind, self.device = hd, kind, device
        self._st = None

    def update(self, image, out=None, update_state=True, stream=None):
        """update(image, update_state).  image: (h, w) or (h, w, 3) float32 / float64, C-contiguous numpy array or
        torch tensor, updated in place; or (h, w, 3) float16, converted into `out` ((h, w, 3) float32, allocated
        when None and returned).  CUDA tensors run on the torch current stream and nothing waits for the GPU."""
        shape = tuple(image.shape)
        dt = _np_dtype(image) if not (_is_torch(image) and str(image.dtype) == "torch.float16") else np.dtype(np.float16)
        if len(shape) == 3 and shape[2] != 3 or len(shape) not in (2, 3):
            raise ValueError("Expected an H x W x 3 array")
        contiguous = image.is_contiguous() if _is_torch(image) else image.flags["C_CONTIGUOUS"]
        if not contiguous:
            raise TypeError("image must be C-contiguous")
        rows, cols = shape[0], shape[1]
        if dt == np.float16 and len(shape) != 3:
            raise ValueError("Expected an H x W x 3 array")
        if dt not in (np.float16, np.float32, np.float64):
            raise TypeError("image must be float32 or float64")
        st = self._st = _stream_for(image, stream, self.device)
        if dt == np.float16:
            if out is None:
                out = _empty(image, shape, np.float32)
            check(lib.ob_image_proc_update(self._h, _capi.OB_IMAGE_RGB_F16, _capi.OB_F32, _ptr(image), _ptr(out),
                                           rows, cols, int(bool(update_state)), st.h))
            return out
        layout = _capi.OB_IMAGE_MONO if len(shape) == 2 else _capi.OB_IMAGE_RGB
        dtype = _capi.OB_F32 if dt == np.float32 else _capi.OB_F64
        check(lib.ob_image_proc_update(self._h, layout, dtype, None, _ptr(image), rows, cols,
                                       int(bool(update_state)), st.h))
        return None

    def state(self, stream=None):
        """Synchronising read of the state: dict with lo, hi, lo_state, hi_state, counter, initialized and
        dark_count (float64 array, BeamUniformityCorrector)."""
        st = stream or self._st or _stream(None, self.device)
        s = _capi.ImageState()
        probe = _capi.ImageState()
        check(lib.ob_image_proc_state(self._h, C.byref(probe), None, 0, st.h))
        dc = np.zeros(max(probe.dark_count_rows, 1), np.float64)
        check(lib.ob_image_proc_state(self._h, C.byref(s), dc.ctypes.data, dc.size, st.h))
        return dict(lo=s.lo, hi=s.hi, lo_state=s.lo_state, hi_state=s.hi_state, counter=s.counter,
                    initialized=bool(s.initialized), dark_count=dc[:s.dark_count_rows])
