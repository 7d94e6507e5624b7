"""ctypes/numpy front-end of the align_clouds oracle (oracle/orc_align_clouds.c, built by oracle/align_clouds.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates the point-cloud align_clouds overloads
(ouster_algorithm/src/align_clouds.cpp:396-1581, 1876-1995, 2601-2651) over the ICP and voxel oracles
(orc_align.c, orc_voxel.c).  `Trace` has the layout of ob_align_clouds_trace (include/ouster_b200.h).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_align_clouds.so")
_SRCS = [os.path.join(_HERE, f) for f in ("orc_align_clouds.c", "orc_align.c", "orc_voxel.c")]

COARSE_YAWS, FINE_YAWS, Z_BINS = 180, 7, 1024
MAX_FINE_BASE, MAX_COARSE_BASE = 481, 241   # base_n at a 60 m bound: 0.25 m and 0.5 m pixels


class Trace(C.Structure):
    _fields_ = [("source_features", C.c_size_t), ("target_features", C.c_size_t),
                ("searched", C.c_int32), ("coarse_index", C.c_int32), ("fine_index", C.c_int32), ("pad", C.c_int32),
                ("bound_m", C.c_double), ("fine_pixel_m", C.c_double), ("coarse_pixel_m", C.c_double),
                ("max_shift_m", C.c_double),
                ("fine_base_n", C.c_int32), ("fine_fft_n", C.c_int32), ("fine_max_shift", C.c_int32),
                ("coarse_base_n", C.c_int32), ("coarse_fft_n", C.c_int32), ("coarse_max_shift", C.c_int32),
                ("coarse_scores", C.c_double * COARSE_YAWS),
                ("fine_z_bins", C.c_int32 * FINE_YAWS), ("fine_dx", C.c_int32 * FINE_YAWS),
                ("fine_dy", C.c_int32 * FINE_YAWS), ("pad2", C.c_int32),
                ("fine_scores", C.c_double * FINE_YAWS),
                ("initial_pose", C.c_double * 16), ("icp_poses", C.c_double * 48),
                ("initial_confidence", C.c_double), ("refined_confidence", C.c_double),
                ("initial_matched", C.c_size_t), ("initial_total", C.c_size_t),
                ("refined_matched", C.c_size_t), ("refined_total", C.c_size_t), ("stage_ms", C.c_double * 5),
                ("target_fine_grid", C.c_void_p), ("target_coarse_grid", C.c_void_p),
                ("target_z_hist", C.c_void_p)]


def trace_dict(t, grids=None):
    """A Trace as plain numpy / Python values; `grids` = (fine, coarse, z_hist) buffers given to the call."""
    d = {name: getattr(t, name) for name, _ in Trace._fields_ if not name.startswith("pad") and not name.endswith(("_grid", "_hist"))}
    for k in ("coarse_scores", "fine_scores", "initial_pose", "icp_poses", "stage_ms"):
        d[k] = np.array(d[k][:], np.float64)
    for k in ("fine_z_bins", "fine_dx", "fine_dy"):
        d[k] = np.array(d[k][:], np.int32)
    d["initial_pose"] = d["initial_pose"].reshape(4, 4)
    d["icp_poses"] = d["icp_poses"].reshape(3, 4, 4)
    if grids is not None:
        fine, coarse, hist = grids
        fb, cb = t.fine_base_n, t.coarse_base_n
        d["target_fine_grid"] = fine[:fb * fb].reshape(fb, fb).copy() if t.searched else None
        d["target_coarse_grid"] = coarse[:cb * cb].reshape(cb, cb).copy() if t.searched else None
        d["target_z_hist"] = hist.copy() if t.searched else None
    return d


def build(force=False):
    """Compile the oracle (gcc); no-op when the .so is up to date."""
    if not force and os.path.exists(_LIB_PATH) and \
            os.path.getmtime(_LIB_PATH) >= max(os.path.getmtime(s) for s in _SRCS):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "align_clouds.mk"])
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
    L.orc_align_clouds_trace_size.restype = i32
    L.orc_align_clouds.argtypes = [vp, vp, sz, vp, vp, sz, vp, i32, vp, C.POINTER(d), C.POINTER(Trace)]
    L.orc_align_clouds.restype = i32
    L.orc_align_clouds_confidence.argtypes = [vp, vp, sz, vp, vp, sz, vp, C.POINTER(sz), C.POINTER(sz)]
    L.orc_align_clouds_confidence.restype = d
    L.orc_align_clouds_features.argtypes = [vp, vp, sz, vp, vp]
    L.orc_align_clouds_features.restype = sz
    assert L.orc_align_clouds_trace_size() == C.sizeof(Trace)
    _lib = L
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rows(a, name):
    a = np.asarray(a)
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError(f"{name} must have shape (N, 3)")
    return np.ascontiguousarray(a, np.float64)


def _check(sp, sn, tp, tn):
    """The reference's checks in its order (align_clouds.cpp:788-803, 856-867)."""
    s = _rows(sp, "source_points")
    ns = None if sn is None else _rows(sn, "source_normals")
    if ns is not None and len(ns) != len(s):
        raise ValueError("source_points and source_normals must have the same number of rows")
    t = _rows(tp, "target_points")
    nt = None if tn is None else _rows(tn, "target_normals")
    if nt is not None and len(nt) != len(t):
        raise ValueError("target_points and target_normals must have the same number of rows")
    if (ns is None) != (nt is None):
        raise ValueError("source_normals and target_normals must both be given or both be omitted")
    return s, ns, t, nt


def align_clouds(source_points, target_points, initial_guess=None, source_normals=None, target_normals=None,
                 compute_confidence=True, grids=False):
    """-> (pose 4x4, confidence, trace dict).  grids: also return the target's raw BEV grids and Z histogram."""
    s, ns, t, nt = _check(source_points, source_normals, target_points, target_normals)
    g = np.eye(4) if initial_guess is None else np.ascontiguousarray(initial_guess, np.float64).reshape(4, 4)
    tr = Trace()
    bufs = None
    if grids:
        bufs = (np.zeros(MAX_FINE_BASE ** 2), np.zeros(MAX_COARSE_BASE ** 2), np.zeros(Z_BINS))
        tr.target_fine_grid, tr.target_coarse_grid, tr.target_z_hist = (b.ctypes.data for b in bufs)
    pose, conf = np.empty((4, 4)), C.c_double(0.0)
    rc = lib().orc_align_clouds(_ptr(s), _ptr(ns), len(s), _ptr(t), _ptr(nt), len(t), _ptr(g),
                                int(bool(compute_confidence)), _ptr(pose), C.byref(conf), C.byref(tr))
    assert rc == 0
    return pose, conf.value, trace_dict(tr, bufs)


def confidence(source_features, target_features, pose, source_normals=None, target_normals=None):
    """xy_matching_confidence of two feature clouds at `pose` -> (confidence, matched, total)."""
    s, t = _rows(source_features, "source"), _rows(target_features, "target")
    ns = None if source_normals is None else _rows(source_normals, "source_normals")
    nt = None if target_normals is None else _rows(target_normals, "target_normals")
    p = np.ascontiguousarray(pose, np.float64).reshape(4, 4)
    m, n = C.c_size_t(0), C.c_size_t(0)
    c = lib().orc_align_clouds_confidence(_ptr(s), _ptr(ns), len(s), _ptr(t), _ptr(nt), len(t), _ptr(p),
                                          C.byref(m), C.byref(n))
    return c, m.value, n.value


def features(points, normals=None):
    """The feature cloud of one input: (points k x 3, normals k x 3 or None)."""
    p = _rows(points, "points")
    n = None if normals is None else _rows(normals, "normals")
    op, on = np.empty((len(p) + 1, 3)), np.empty((len(p) + 1, 3))
    k = lib().orc_align_clouds_features(_ptr(p), _ptr(n), len(p), _ptr(op), _ptr(on))
    return op[:k].copy(), (on[:k].copy() if n is not None else None)
