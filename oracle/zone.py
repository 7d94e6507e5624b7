"""ctypes/numpy front-end of the zone-monitoring oracle (oracle/orc_zone.c, built by oracle/zone.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates Zone::render (ouster_core/src/zone.cpp:63-135) with
Mesh::closest_and_farthest_intersections and its bounding sphere (mesh.cpp:41-60, 249-294), Triangle::intersect
(triangle.cpp:19-50), the BeamConfig LUTs (beam_config.cpp:14-45), and EmulatedZoneMon's counts and trigger
counters (python/src/ouster/sdk/core/zone_common.py:47-105).
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import oracle as _orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_zone.so")
_SRC = os.path.join(_HERE, "orc_zone.c")

RANGE_OVERFLOW = "Zone::render: range overflow"


def build(force=False):
    """Compile the oracle (gcc); no-op when the .so is up to date."""
    if not force and os.path.exists(_LIB_PATH) and os.path.getmtime(_LIB_PATH) >= os.path.getmtime(_SRC):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "zone.mk"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        build()
    L = C.CDLL(_LIB_PATH)
    vp, sz, u32 = C.c_void_p, C.c_size_t, C.c_uint32
    L.orc_tri_intersect.argtypes = [vp, vp, vp]
    L.orc_tri_intersect.restype = C.c_float
    L.orc_bounding_sphere.argtypes = [vp, sz, vp]
    L.orc_closest_and_farthest.argtypes = [vp, sz, vp, vp, vp]
    L.orc_closest_and_farthest.restype = C.c_int
    L.orc_zone_render.argtypes = [vp, sz, vp, vp, sz, sz, u32, vp, vp, C.POINTER(u32)]
    L.orc_zone_render.restype = C.c_int
    L.orc_zone_counts.argtypes = [vp, vp, vp, sz, u32, vp, vp]
    L.orc_zone_trigger.argtypes = [C.c_int, u32, u32, u32, C.POINTER(u32), C.POINTER(u32)]
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _tris(t):
    t = np.ascontiguousarray(t, np.float32).reshape(-1, 9)
    return t


def tri_intersect(tri, offset, direction):
    """Triangle(v0, v1, v2).intersect(Ray{offset, direction}) (float32 inputs)."""
    t = _tris(tri)
    o = np.ascontiguousarray(offset, np.float32)
    d = np.ascontiguousarray(direction, np.float32)
    return float(lib().orc_tri_intersect(_ptr(t), _ptr(o), _ptr(d)))


def bounding_sphere(tris):
    """Mesh(tris).bounding_sphere(): (centroid float32[3], radius float32)."""
    t = _tris(tris)
    out = np.empty(4, np.float32)
    lib().orc_bounding_sphere(_ptr(t), len(t), _ptr(out))
    return out[:3].copy(), out[3]


def closest_and_farthest(tris, offset, direction):
    """Mesh(tris).closest_and_farthest_intersections(Ray): (bool, (near, far) float32)."""
    t = _tris(tris)
    o = np.ascontiguousarray(offset, np.float32)
    d = np.ascontiguousarray(direction, np.float32)
    b = np.zeros(2, np.float32)
    ok = lib().orc_closest_and_farthest(_ptr(t), len(t), _ptr(o), _ptr(d), _ptr(b))
    return bool(ok), (b[0], b[1])


def scale_translation(m):
    """beam_config.cpp:14-20"""
    r = np.array(m, np.float64).reshape(4, 4).copy()
    r[:3, 3] *= 1000
    return r


def beam_luts(meta, sensor_to_body=None):
    """BeamConfig's two LUTs (beam_config.cpp:37-45) from sensor metadata (w, h, beam_to_lidar_transform,
    lidar_to_sensor_transform, beam_azimuth_angles, beam_altitude_angles): (body (direction, offset) or None,
    sensor (direction, offset)), each (h*w, 3) float64."""
    w, h = meta["w"], meta["h"]
    b2l, l2s = meta["beam_to_lidar_transform"], np.array(meta["lidar_to_sensor_transform"], np.float64).reshape(4, 4)
    az, alt = meta["beam_azimuth_angles"], meta["beam_altitude_angles"]
    sensor = _orc.make_xyz_lut(w, h, 0.001, b2l, l2s, az, alt)
    body = None
    if sensor_to_body is not None:
        body = _orc.make_xyz_lut(w, h, 0.001, b2l, scale_translation(sensor_to_body) @ l2s, az, alt)
    return body, sensor


def render(tris, direction, offset, h, w, point_count=1):
    """Zone::render's loop over one LUT: (near_mm, far_mm uint32 (h, w), pixels_with_intersections).
    Raises RuntimeError with the reference's texts for a range overflow and a too-small area."""
    t = _tris(tris)
    d = np.ascontiguousarray(direction, np.float64).reshape(-1)
    o = np.ascontiguousarray(offset, np.float64).reshape(-1)
    assert d.size == o.size == h * w * 3
    near, far = np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint32)
    px = C.c_uint32(0)
    rc = lib().orc_zone_render(_ptr(t), len(t), _ptr(d), _ptr(o), h, w, int(point_count), _ptr(near), _ptr(far),
                               C.byref(px))
    if rc == -1:
        raise RuntimeError(RANGE_OVERFLOW)
    if rc == -2:
        raise RuntimeError(f"Zone: area of rendered zone ({px.value}) is smaller than point_count ({point_count}) "
                           "specified in zone.")
    return near, far, px.value


def counts(range_img, near, far, live_index=0, bitmask=None):
    """_calc_counts for one live zone: dict of count, occlusion_count, invalid_count, min_range, max_range,
    mean_range; ORs 1 << live_index into `bitmask` (uint32, C-contiguous) where the zone triggers."""
    r = np.ascontiguousarray(range_img, np.uint32)
    n = np.ascontiguousarray(near, np.uint32)
    f = np.ascontiguousarray(far, np.uint32)
    assert r.size == n.size == f.size
    out = np.zeros(6, np.uint32)
    if bitmask is not None:
        assert bitmask.dtype == np.uint32 and bitmask.flags["C_CONTIGUOUS"] and bitmask.size == r.size
    lib().orc_zone_counts(_ptr(r), _ptr(n), _ptr(f), r.size, int(live_index),
                          None if bitmask is None else _ptr(bitmask), _ptr(out))
    keys = ("count", "occlusion_count", "invalid_count", "min_range", "max_range", "mean_range")
    return {k: int(v) for k, v in zip(keys, out)}


def trigger(mode, point_count, frame_count, count, triggers, alerts):
    """calc_triggers' counters for one zone: -> (triggers, alerts)."""
    t, a = C.c_uint32(triggers), C.c_uint32(alerts)
    lib().orc_zone_trigger(int(mode), int(point_count), int(frame_count), int(count), C.byref(t), C.byref(a))
    return t.value, a.value
