"""ctypes/numpy front-end of the cloud-to-cloud ICP oracle (oracle/orc_align.c, built by oracle/align.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates point_to_point_align / point_to_plane_align and the
SpatialHashGrid3D they search (ouster_algorithm/src/align_clouds.cpp:146-235, 1590-1874), PoseV::exp
(ouster_core/src/transform_vector.cpp:40-104) and the Eigen pieces they use (JacobiSVD<Matrix3d>, LDLT 6x6).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_align.so")
_SRC = os.path.join(_HERE, "orc_align.c")

ERRORS = {-1: "max_corr_dist must be finite and greater than zero",
          -2: "max_normal_angle_deg must be finite and in [0, 180]",
          -3: "source_points and source_normals must have the same number of rows",
          -4: "target_points and target_normals must have the same number of rows"}


def build(force=False):
    """Compile the oracle (gcc); no-op when the .so is up to date."""
    if not force and os.path.exists(_LIB_PATH) and os.path.getmtime(_LIB_PATH) >= os.path.getmtime(_SRC):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "align.mk"])
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
    L.orc_cell_coord.argtypes = [d, d]
    L.orc_cell_coord.restype = C.c_int64
    L.orc_median_abs.argtypes = [vp, sz]
    L.orc_median_abs.restype = d
    L.orc_cloud_nearest.argtypes = [vp, vp, sz, d, vp, sz, d, vp]
    L.orc_svd3.argtypes = [vp, vp, vp, vp]
    L.orc_svd3.restype = i32
    L.orc_ldlt6.argtypes = [vp, vp, vp]
    L.orc_ldlt6.restype = i32
    L.orc_posev_exp.argtypes = [vp, vp]
    L.orc_point_to_point_align.argtypes = [vp, sz, vp, sz, vp, d, vp, C.POINTER(i32)]
    L.orc_point_to_point_align.restype = i32
    L.orc_point_to_plane_align.argtypes = [vp, sz, vp, sz, vp, sz, vp, sz, vp, d, d, vp, C.POINTER(i32)]
    L.orc_point_to_plane_align.restype = i32
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _rows(a):
    a = np.ascontiguousarray(a, np.float64)
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError("expected an Nx3 array")
    return a


def _guess(g):
    return np.eye(4) if g is None else np.ascontiguousarray(g, np.float64).reshape(4, 4)


def cell_coord(v, inv_cell_size):
    """static_cast<int64_t>(std::floor(v * inv)) as x86 evaluates it (INT64_MIN for NaN / out of range)."""
    return int(lib().orc_cell_coord(float(v), float(inv_cell_size)))


def median_abs(v):
    v = np.ascontiguousarray(v, np.float64).reshape(-1)
    return float(lib().orc_median_abs(_ptr(v), len(v)))


def cloud_nearest(target, queries, cell_size, max_dist_sq, target_normals=None):
    """SpatialHashGrid3D(target[, target_normals], cell_size).nearest(target, q, max_dist_sq) per query row: int32."""
    t, q = _rows(target), _rows(queries)
    nrm = None if target_normals is None else _rows(target_normals)
    out = np.empty(len(q), np.int32)
    lib().orc_cloud_nearest(_ptr(t), None if nrm is None else _ptr(nrm), len(t), float(cell_size), _ptr(q), len(q),
                            float(max_dist_sq), _ptr(out))
    return out


def svd3(a):
    """Eigen::JacobiSVD<Matrix3d>(a, ComputeFullU | ComputeFullV): (U, singular values decreasing, V, info)."""
    a = np.ascontiguousarray(a, np.float64).reshape(3, 3)
    u, s, v = np.empty((3, 3)), np.empty(3), np.empty((3, 3))
    info = lib().orc_svd3(_ptr(a), _ptr(u), _ptr(s), _ptr(v))
    return u, s, v, info


def ldlt6(a, b):
    """Eigen's LDLT of a 6x6 (lower triangle read): (solve(b), info 0 = Success / 1 = NumericalIssue)."""
    a = np.ascontiguousarray(a, np.float64).reshape(6, 6)
    b = np.ascontiguousarray(b, np.float64).reshape(6)
    x = np.empty(6)
    info = lib().orc_ldlt6(_ptr(a), _ptr(b), _ptr(x))
    return x, info


def posev_exp(v):
    """PoseV(v).exp() as a 4x4, v = (rotation vector, translation)."""
    v = np.ascontiguousarray(v, np.float64).reshape(6)
    m = np.empty((4, 4))
    lib().orc_posev_exp(_ptr(v), _ptr(m))
    return m


def point_to_point_align(source, target, initial_guess=None, max_corr_dist=0.25):
    """-> (4x4 float64, iterations that reached the solve)."""
    s, t, g = _rows(source), _rows(target), _guess(initial_guess)
    out, it = np.empty((4, 4)), C.c_int(0)
    rc = lib().orc_point_to_point_align(_ptr(s), len(s), _ptr(t), len(t), _ptr(g), float(max_corr_dist), _ptr(out),
                                        C.byref(it))
    if rc:
        raise ValueError(ERRORS[rc])
    return out, it.value


def point_to_plane_align(source, target, source_normals, target_normals, initial_guess=None, max_corr_dist=0.25,
                         max_normal_angle_deg=20.0):
    """-> (4x4 float64, iterations that reached the solve)."""
    s, t, g = _rows(source), _rows(target), _guess(initial_guess)
    sn, tn = _rows(source_normals), _rows(target_normals)
    out, it = np.empty((4, 4)), C.c_int(0)
    rc = lib().orc_point_to_plane_align(_ptr(s), len(s), _ptr(t), len(t), _ptr(sn), len(sn), _ptr(tn), len(tn),
                                        _ptr(g), float(max_corr_dist), float(max_normal_angle_deg), _ptr(out),
                                        C.byref(it))
    if rc:
        raise ValueError(ERRORS[rc])
    return out, it.value
