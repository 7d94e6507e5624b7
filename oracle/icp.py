"""ctypes/numpy front-end of the frame-to-map registration oracle (oracle/orc_icp.c, built by oracle/icp.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates VoxelHashMap3d (ouster_core/src/voxel_hash_map.cpp:14-247),
ICPRegistration / build_linear_system (ouster_mapping/src/icp_registration.cpp) and the Sophus / Eigen pieces they
use.  Voxels come out in creation order (DESIGN 9).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_icp.so")
_SRC = os.path.join(_HERE, "orc_icp.c")
DBL_MAX = float(np.finfo(np.float64).max)


def build(force=False):
    """Compile the registration oracle (gcc); no-op when the .so is up to date."""
    if not force and os.path.exists(_LIB_PATH) and os.path.getmtime(_LIB_PATH) >= os.path.getmtime(_SRC):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "icp.mk"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        build()
    L = C.CDLL(_LIB_PATH)
    vp, sz, i32, d = C.c_void_p, C.c_size_t, C.c_int, C.c_double
    L.orc_map_create.argtypes = [d, d, sz, sz, C.POINTER(vp)]
    L.orc_map_create.restype = i32
    L.orc_map_destroy.argtypes = [vp]
    L.orc_map_clear.argtypes = [vp]
    L.orc_map_add_points.argtypes = [vp, vp, sz]
    L.orc_map_remove_far.argtypes = [vp, vp, vp]
    L.orc_map_remove_far.restype = sz
    L.orc_map_size.argtypes = [vp, C.POINTER(sz)]
    L.orc_map_size.restype = sz
    L.orc_map_point_cloud.argtypes = [vp, vp]
    L.orc_map_point_cloud.restype = sz
    L.orc_map_closest.argtypes = [vp, vp, d, vp]
    L.orc_map_closest.restype = d
    L.orc_linear_system.argtypes = [vp, vp, sz, d, vp, vp]
    L.orc_ldlt_solve6.argtypes = [vp, vp, vp]
    L.orc_se3_exp.argtypes = [vp, vp]
    L.orc_icp_align.argtypes = [vp, vp, sz, d, d, i32, d, vp]
    L.orc_icp_align.restype = i32
    L.orc_cull_threshold.argtypes = [d, d]
    L.orc_cull_threshold.restype = C.c_int32
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _rows(points):
    p = np.ascontiguousarray(points, np.float64)
    if p.ndim != 2 or p.shape[1] != 3:
        raise ValueError("add_points expects an Nx3 array")
    return p


class VoxelHashMap3d:
    """VoxelHashMap3d(voxel_size, max_distance=100, max_points_per_voxel=20, min_pts_threshold=1), first_n_point."""

    def __init__(self, voxel_size, max_distance=100.0, max_points_per_voxel=20, min_pts_threshold=1):
        h = C.c_void_p()
        rc = lib().orc_map_create(float(voxel_size), float(max_distance), int(max_points_per_voxel),
                                  int(min_pts_threshold), C.byref(h))
        if rc:
            raise ValueError({-1: "max_points_per_voxel must be greater than 0", -2: "voxel_size must be greater than 0",
                              -3: "max_distance must be greater than 0"}[rc])
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.orc_map_destroy(self._h)
            self._h = None

    def clear(self):
        lib().orc_map_clear(self._h)

    @property
    def empty(self):
        return self.size()[0] == 0

    def size(self):
        """(live voxels, stored points)"""
        pts = C.c_size_t(0)
        v = lib().orc_map_size(self._h, C.byref(pts))
        return v, pts.value

    def add_points(self, points):
        p = _rows(points)
        lib().orc_map_add_points(self._h, _ptr(p), len(p))

    def point_cloud(self):
        out = np.empty((self.size()[1], 3))
        k = lib().orc_map_point_cloud(self._h, _ptr(out))
        return out[:k]

    def remove_voxels_far_from_location(self, origin):
        o = np.ascontiguousarray(origin, np.float64).reshape(3)
        lib().orc_map_remove_far(self._h, _ptr(o), None)

    def extract_voxels_far_from_location(self, origin):
        o = np.ascontiguousarray(origin, np.float64).reshape(3)
        out = np.empty((self.size()[1], 3))
        k = lib().orc_map_remove_far(self._h, _ptr(o), _ptr(out))
        return out[:k]

    def get_closest_neighbor(self, point, max_distance_sq=DBL_MAX):
        q = np.ascontiguousarray(point, np.float64).reshape(3)
        nb = np.empty(3)
        d2 = lib().orc_map_closest(self._h, _ptr(q), float(max_distance_sq), _ptr(nb))
        return nb, d2

    def get_closest_neighbors(self, points, max_distance_sq=DBL_MAX):
        p = _rows(points)
        nb = np.empty_like(p)
        d2 = np.empty(len(p))
        for i in range(len(p)):
            d2[i] = lib().orc_map_closest(self._h, _ptr(p[i]), float(max_distance_sq), _ptr(nb[i]))
        return nb, d2


def cull_threshold(max_distance, voxel_size):
    """(ceil(max_distance / voxel_size) + 1)^2 in wrapping int32 arithmetic."""
    return int(lib().orc_cull_threshold(float(max_distance), float(voxel_size)))


def build_linear_system(source, target, kernel_scale):
    """build_linear_system(correspondences, kernel_scale) -> (jtj [6, 6] lower triangle, jtr [6])."""
    s = np.ascontiguousarray(source, np.float64).reshape(-1, 3)
    t = np.ascontiguousarray(target, np.float64).reshape(-1, 3)
    jtj, jtr = np.empty((6, 6)), np.empty(6)
    lib().orc_linear_system(_ptr(s), _ptr(t), len(s), float(kernel_scale), _ptr(jtj), _ptr(jtr))
    return jtj, jtr


def ldlt_solve(a, b):
    """Eigen's a.ldlt().solve(b) for a 6x6 matrix (lower triangle read)."""
    a = np.ascontiguousarray(a, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    x = np.empty(6)
    lib().orc_ldlt_solve6(_ptr(a), _ptr(b), _ptr(x))
    return x


def se3_exp(a):
    """Sophus::SE3d::exp(a).matrix(), a = (translation part, rotation part)."""
    a = np.ascontiguousarray(a, np.float64)
    m = np.empty((4, 4))
    lib().orc_se3_exp(_ptr(a), _ptr(m))
    return m


def align_points_to_map(frame, voxel_map, max_distance, kernel_scale, max_num_iterations=50,
                        convergence_criterion=1e-4):
    """ICPRegistration::align_points_to_map -> (4x4 float64, iterations run)."""
    f = _rows(frame)
    m = np.empty((4, 4))
    it = lib().orc_icp_align(voxel_map._h, _ptr(f), len(f), float(max_distance), float(kernel_scale),
                             int(max_num_iterations), float(convergence_criterion), _ptr(m))
    return m, it
