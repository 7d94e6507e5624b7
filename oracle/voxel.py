"""ctypes/numpy front-end of the voxel-downsampling oracle (oracle/orc_voxel.c, built by oracle/voxel.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates ouster_core/src/voxel_hash_map.cpp:262-393 and
ouster_algorithm/src/voxel_downsample.cpp:21-57.  Voxels come out in first-appearance order (DESIGN 9).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_voxel.so")
_SRC = os.path.join(_HERE, "orc_voxel.c")

FIRST_N_POINT, AVERAGE_POINT, RANDOM = 0, 1, 2     # core::VoxelDownsampleStrategy


def build(force=False):
    """Compile the voxel oracle (gcc); no-op when the .so is up to date."""
    if not force and os.path.exists(_LIB_PATH) and os.path.getmtime(_LIB_PATH) >= os.path.getmtime(_SRC):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "voxel.mk"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        build()
    L = C.CDLL(_LIB_PATH)
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    L.orc_voxel_coord.argtypes = [C.c_double]
    L.orc_voxel_coord.restype = C.c_int32
    L.orc_voxel_downsample.argtypes = [vp, sz, C.c_double, vp, vp]
    L.orc_voxel_downsample.restype = sz
    L.orc_voxel_downsample_xd.argtypes = [vp, sz, sz, C.c_double, sz, sz, i32, vp, vp, C.POINTER(sz)]
    L.orc_voxel_downsample_xd.restype = i32
    L.orc_voxel_downsample_with_normals.argtypes = [vp, vp, sz, C.c_double, vp, vp, vp, C.POINTER(sz)]
    L.orc_voxel_downsample_with_normals.restype = i32
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def voxel_coord(v):
    """int(floor(v)) as x86 cvttsd2si gives it: INT32_MIN for NaN and out-of-range values."""
    return int(lib().orc_voxel_coord(float(v)))


def voxel_downsample(points, voxel_size):
    """core::voxel_downsample(frame, voxel_size) -> (points [m, 3] float64, indices [m] uint32)."""
    p = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
    out = np.empty_like(p)
    idx = np.empty(len(p), np.uint32)
    m = lib().orc_voxel_downsample(_ptr(p), len(p), float(voxel_size), _ptr(out), _ptr(idx))
    return out[:m].copy(), idx[:m].copy()


def voxel_downsample_xd(frame, voxel_size, max_points_per_voxel=1, min_pts_threshold=1, strategy=RANDOM,
                        with_indices=False, name="voxel_downsample_xd"):
    """core::voxel_downsample_xd (and _3d with name="voxel_downsample_3d"): [n, cols] -> [m, cols] float64
    (and the source index of every row with with_indices=True).  ValueError texts of the reference."""
    f = np.ascontiguousarray(frame, np.float64)
    n, cols = f.shape
    out = np.empty((n, cols), np.float64)
    idx = np.empty(n, np.uint32)
    m = C.c_size_t(0)
    rc = lib().orc_voxel_downsample_xd(_ptr(f), n, cols, float(voxel_size), int(max_points_per_voxel),
                                       int(min_pts_threshold), int(strategy), _ptr(out), _ptr(idx), C.byref(m))
    msgs = {-1: "max_points_per_voxel must be greater than 0", -2: "voxel_size must be greater than 0",
            -3: f"{name}: frame must have at least 3 columns", -4: f"{name}: unknown strategy"}
    if rc:
        raise ValueError(msgs[rc])
    k = m.value
    return (out[:k].copy(), idx[:k].copy()) if with_indices else out[:k].copy()


def voxel_downsample_with_normals(points, normals, voxel_size, with_indices=False):
    """algorithm::voxel_downsample_with_normals -> (points [m, 3], normals [m, 3]) float64."""
    p = np.ascontiguousarray(points, np.float64)
    q = np.ascontiguousarray(normals, np.float64)
    if p.ndim != 2 or q.ndim != 2 or p.shape[1] != 3 or q.shape[1] != 3:
        raise ValueError("voxel_downsample_with_normals expects Nx3 inputs")
    if p.shape[0] != q.shape[0]:
        raise ValueError("voxel_downsample_with_normals points/normals size mismatch")
    n = p.shape[0]
    op, on = np.empty((n, 3)), np.empty((n, 3))
    idx = np.empty(n, np.uint32)
    m = C.c_size_t(0)
    if lib().orc_voxel_downsample_with_normals(_ptr(p), _ptr(q), n, float(voxel_size), _ptr(op), _ptr(on), _ptr(idx),
                                               C.byref(m)):
        raise ValueError("voxel_downsample_with_normals voxel_size must be > 0")
    k = m.value
    res = (op[:k].copy(), on[:k].copy())
    return res + (idx[:k].copy(),) if with_indices else res
