"""ctypes/numpy front-end of the ground-segmentation oracle (oracle/orc_ground.c, built by oracle/ground.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates impl::get_ground_mask and the ground model passes of
ouster_algorithm/src/ground_seg.cpp:179-1314.  Normals, when the frame carries none, come from the normals oracle
(oracle.normals) on the dewarped points with per-column sensor origins, as get_ground_mask_into does
(ground_seg.cpp:1195-1250).
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_ground.so")
_SRCS = [os.path.join(_HERE, "orc_ground.c")]

# passes of the model, in order; run(stop=...) returns the model after that pass
STAGES = ("cells", "fill1", "smooth1", "prune", "fill2", "smooth2", "components", "fill3")
FINAL = len(STAGES) - 1

ERR_SENSOR_INFO = "frame.sensor_info is required for get_ground_mask"
ERR_RANGE = "frame must contain RANGE field for get_ground_mask"
ERR_GRID_SIZE = "GroundSegConfig.grid_size must be > 0"


class _Frame(C.Structure):
    _fields_ = [("h", C.c_int), ("w", C.c_int), ("n_returns", C.c_int), ("pad", C.c_int),
                ("range", C.POINTER(C.c_void_p)), ("status", C.c_void_p), ("dir", C.c_void_p),
                ("off", C.c_void_p), ("poses", C.c_void_p), ("normals", C.c_void_p * 2), ("grid_size", C.c_double)]


class _Model(C.Structure):
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("fallback_z", C.c_double),
                ("footprint_bound", C.c_double), ("rows", C.c_int32), ("cols", C.c_int32), ("valid", C.c_int32),
                ("has_columns", C.c_int32)]


def build(force=False):
    """Compile the oracle (gcc); no-op when the .so is up to date."""
    if (not force and os.path.exists(_LIB_PATH)
            and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in _SRCS)):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "ground.mk"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    build()
    L = C.CDLL(_LIB_PATH)
    vp = C.c_void_p
    L.orc_ground_run.argtypes = [C.POINTER(_Frame), C.c_int, vp, C.POINTER(_Model), vp, vp, vp, vp, vp]
    L.orc_ground_run.restype = None
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data if a is not None else None


def dewarped_points(rng, direction, offset, poses):
    """cartesianT then dewarp (double): (H, W, 3)."""
    h, w = rng.shape
    pts = orc.cartesian(rng, np.asarray(direction, np.float64).reshape(-1, 3),
                        np.asarray(offset, np.float64).reshape(-1, 3)).reshape(h, w, 3)
    return orc.dewarp(pts, np.asarray(poses, np.float64).reshape(w, 16)).reshape(h, w, 3)


def sensor_origins(poses, sensor_to_body):
    """(pose_c * sensor_to_body).translation per column, summed as ((a0 + a1) + a2) + a3: W x 3."""
    p = np.asarray(poses, np.float64).reshape(-1, 4, 4)
    t = np.asarray(sensor_to_body, np.float64).reshape(4, 4)[:, 3]
    acc = p[:, :3, 0] * t[0]
    for k in range(1, 4):
        acc = acc + p[:, :3, k] * t[k]
    return np.ascontiguousarray(acc)


def computed_normals(ranges, direction, offset, poses, sensor_to_body):
    """The normals get_ground_mask computes when the frame has no NORMALS field: one (H, W, 3) per model return."""
    origins = sensor_origins(poses, sensor_to_body)
    p0 = dewarped_points(ranges[0], direction, offset, poses)
    if len(ranges) >= 2:
        p1 = dewarped_points(ranges[1], direction, offset, poses)
        n0, n1 = orc.normals(p0, ranges[0], p1, ranges[1], sensor_origins_xyz=origins)
        return [n0, n1]
    return [orc.normals(p0, ranges[0], sensor_origins_xyz=origins)]


def run(ranges, status, direction, offset, poses, normals=None, grid_size=0.5, stop=FINAL):
    """One frame through the oracle.  ranges: list of (H, W) uint32 per return; normals: None or a list of (H, W, 3)
    (entries may be None) for the first two returns.  -> (masks list of (H, W) uint8 (None unless stop == FINAL),
    model dict, grids dict of (rows, cols) arrays or None when the model has no grid)."""
    ranges = [np.ascontiguousarray(r, np.uint32) for r in ranges]
    h, w = ranges[0].shape
    st = np.ascontiguousarray(status, np.uint32).reshape(w)
    d = np.ascontiguousarray(direction, np.float64).reshape(h * w, 3)
    o = np.ascontiguousarray(offset, np.float64).reshape(h * w, 3)
    ps = np.ascontiguousarray(poses, np.float64).reshape(w, 16)
    nrm = [None, None]
    for i, n in enumerate((normals or [])[:2]):
        if n is not None and i < len(ranges):
            nrm[i] = np.ascontiguousarray(n, np.float64).reshape(h * w, 3)
    rp = (C.c_void_p * len(ranges))(*[r.ctypes.data for r in ranges])
    f = _Frame(h, w, len(ranges), 0, C.cast(rp, C.POINTER(C.c_void_p)), _ptr(st), _ptr(d), _ptr(o), _ptr(ps),
               (C.c_void_p * 2)(_ptr(nrm[0]), _ptr(nrm[1])), float(grid_size))
    m = _Model()
    L = lib()
    L.orc_ground_run(C.byref(f), int(stop), None, C.byref(m), None, None, None, None, None)
    n = int(m.rows) * int(m.cols)
    grids = None
    masks = [np.zeros((h, w), np.uint8) for _ in ranges]
    mp = (C.c_void_p * len(ranges))(*[x.ctypes.data for x in masks])
    if n > 0:
        grids = {"valid": np.zeros(n, np.uint8), "obstacle": np.zeros(n, np.uint8), "floor_z": np.zeros(n),
                 "height": np.zeros(n), "roughness": np.zeros(n)}
        L.orc_ground_run(C.byref(f), int(stop), C.cast(mp, C.c_void_p), C.byref(m), *[_ptr(grids[k]) for k in (
            "valid", "obstacle", "floor_z", "height", "roughness")])
        grids = {k: v.reshape(m.rows, m.cols) for k, v in grids.items()}
    else:
        L.orc_ground_run(C.byref(f), int(stop), C.cast(mp, C.c_void_p), C.byref(m), None, None, None, None, None)
    model = {k: getattr(m, k) for k, _ in _Model._fields_}
    return (masks if stop == FINAL else None), model, grids


def get_ground_mask(frame, grid_size=0.5):
    """impl::get_ground_mask on a frame given as a dict: "sensor_info" (None or a dict with "sensor_to_body"),
    "fields" (RANGE, RANGE2, ..., optional NORMALS / NORMALS2 float32 (H, W, 3)), "status", "poses" (W x 4 x 4),
    "direction" / "offset" (the use_extrinsics LUT, H*W x 3).  -> list of (H, W) uint8 masks, one per return
    present; ValueError with the reference's texts."""
    if frame.get("sensor_info") is None:
        raise ValueError(ERR_SENSOR_INFO)
    fields = frame["fields"]
    if "RANGE" not in fields:
        raise ValueError(ERR_RANGE)
    ranges = [fields["RANGE"]]
    for k in range(2, int(frame["sensor_info"].get("num_returns", 2)) + 1):
        if "RANGE%d" % k not in fields:
            break
        ranges.append(fields["RANGE%d" % k])
    if "NORMALS" in fields:
        normals = [fields["NORMALS"].astype(np.float64)]
        if len(ranges) >= 2 and "NORMALS2" in fields:
            normals.append(fields["NORMALS2"].astype(np.float64))
    elif np.any(np.asarray(frame["status"]) & 1):
        normals = computed_normals(ranges, frame["direction"], frame["offset"], frame["poses"],
                                   frame["sensor_info"]["sensor_to_body"])
    else:
        normals = None
    masks, _, _ = run(ranges, frame["status"], frame["direction"], frame["offset"], frame["poses"], normals,
                      grid_size)
    return masks


def check_grid_size(grid_size):
    """GroundSegEngine::create's check."""
    if not np.isfinite(grid_size) or grid_size <= 0.0:
        raise ValueError(ERR_GRID_SIZE)
