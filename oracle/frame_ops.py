"""ctypes/numpy front-end of the frame operations oracle (oracle/orc_frame_ops.c, built by oracle/frame_ops.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py.  `Frame` is a plain numpy stand-in for the reference's
LidarFrame: named fields with a ChanFieldType tag and a FieldClass, a shift table and body_to_world.  The functions
restate ouster_core/src/frame_ops.cpp and python/src/ouster/sdk/core/frame_ops.py in the reference's order of
operations: field selection, the per-type visit (skips and the dimension error), the mask built before any write,
filter_uv "v" as destagger / mask / stagger.  Each call first validates everything, as the GPU path does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_frame_ops.so")
_SRCS = [os.path.join(_HERE, "orc_frame_ops.c")]

PIXEL_FIELD, COLUMN_FIELD, PACKET_FIELD, FRAME_FIELD = 1, 2, 3, 4
HANDLED = set(range(1, 11))
TAG_NP = {1: np.uint8, 2: np.uint16, 3: np.uint32, 4: np.uint64, 5: np.int8, 6: np.int16, 7: np.int32,
          8: np.int64, 9: np.float32, 10: np.float64, 12: np.uint16}
DIMS_MSG = ("Field: Eigen array conversion failed due to dimension mismatch. Underlying data has {} dimensions "
            "but must have 2 dimensions.")
SOURCE_MSG = "filter_field requires a pixel field with shape (h, w) to build a mask"
SECOND_RETURN = {"RANGE2", "SIGNAL2", "REFLECTIVITY2", "FLAGS2"}


def build(force=False):
    """Compile the oracle (gcc); no-op when the .so is up to date."""
    if not force and os.path.exists(_LIB_PATH) and \
            all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in _SRCS):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "frame_ops.mk"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp, sz, d, i = C.c_void_p, C.c_size_t, C.c_double, C.c_int
        for name, args in (("orc_fo_clip", [vp, i, sz, d, d, d]), ("orc_fo_filter_mask", [vp, vp, i, sz, d, d]),
                           ("orc_fo_apply_mask", [vp, i, sz, vp, d]), ("orc_fo_uv_v_mask", [vp, vp, sz, sz, sz, sz]),
                           ("orc_fo_uv_v_literal", [vp, i, sz, vp, sz, sz, sz, sz, d]),
                           ("orc_fo_xyz_mask_f64", [vp, vp, sz, i, d, d]),
                           ("orc_fo_xyz_mask_f32", [vp, vp, sz, i, d, d])):
            f = getattr(L, name)
            f.argtypes = args
            f.restype = i if not name.startswith("orc_fo_uv_v_mask") and "xyz" not in name else None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data


class Frame:
    """fields: {name: (array, tag, field_class)}; pixel arrays are (h, w[, k])."""

    def __init__(self, h, w, shifts=None, sensor_info=None):
        self.h, self.w = h, w
        self.shifts = np.zeros(h, np.int32) if shifts is None else np.asarray(shifts, np.int32)
        self.sensor_info = sensor_info
        self._f = {}
        self.body_to_world = np.tile(np.eye(4), (w, 1, 1))
        self.headers = {}

    def add(self, name, array, tag=None, field_class=PIXEL_FIELD):
        a = np.ascontiguousarray(array)
        if tag is None:
            tag = {np.dtype(v): k for k, v in TAG_NP.items() if k != 12}[a.dtype]
        self._f[name] = (a, tag, field_class)
        return a

    @property
    def fields(self):
        return list(self._f)

    def has_field(self, name):
        return name in self._f

    def field(self, name):
        return self._f[name][0]

    def tag(self, name):
        return self._f[name][1]

    def field_class(self, name):
        return self._f[name][2]

    def copy(self):
        out = Frame(self.h, self.w, self.shifts.copy(), self.sensor_info)
        for n, (a, t, c) in self._f.items():
            out._f[n] = (a.copy(), t, c)
        out.body_to_world = self.body_to_world.copy()
        out.headers = {k: np.copy(v) for k, v in self.headers.items()}
        return out


def check_invalid(frame, names, invalid):
    """The GPU path's refusal where static_cast<T>(invalid) is undefined (DESIGN §9)."""
    inv = float(invalid)
    for n in names:
        t = frame.tag(n)
        if t in HANDLED and np.dtype(TAG_NP[t]).kind in "iu":
            info = np.iinfo(TAG_NP[t])
            if not np.isfinite(inv) or not (info.min <= np.trunc(inv) <= info.max) or \
                    (t in (4, 8) and np.trunc(inv) >= 2.0 ** (64 if t == 4 else 63)):
                raise ValueError("invalid value cannot be represented in the field's type")


def resolve_pixel_fields(frame, filtered_fields, python=False):
    """resolve_pixel_fields (frame_ops.cpp:19-62) / _resolve_pixel_fields (frame_ops.py:17-39)."""
    requested = list(filtered_fields) if filtered_fields is not None else frame.fields
    present = [f for f in requested if frame.has_field(f)]
    non_pixel = [f for f in present if frame.field_class(f) != PIXEL_FIELD]
    if filtered_fields is not None and non_pixel:
        if python:
            raise ValueError(f"Only PIXEL_FIELD frame fields are supported here; requested non-pixel fields: "
                             f"{non_pixel}")
        raise ValueError("Only PIXEL_FIELD frame fields are supported here; requested non-pixel fields: ["
                         + ", ".join(non_pixel) + "]")
    return [f for f in present if frame.field_class(f) == PIXEL_FIELD]


def _visited(frame, names):
    """impl::visit_field_2d: handled types that are (h, w); the dimension error for the others; skips."""
    out = []
    for n in names:
        if frame.tag(n) not in HANDLED:
            continue
        a = frame.field(n)
        if a.ndim != 2:
            raise ValueError(DIMS_MSG.format(a.ndim))
        out.append(n)
    return out


def clip(frame, fields, lower, upper, invalid=0):
    names = _visited(frame, resolve_pixel_fields(frame, list(fields) if fields else None))
    check_invalid(frame, names, invalid)
    for n in names:
        a = frame.field(n)
        assert lib().orc_fo_clip(_p(a), frame.tag(n), a.size, lower, upper, float(invalid)) == 0


def _apply(frame, names, mask, invalid):
    for n in names:
        a = frame.field(n)
        assert lib().orc_fo_apply_mask(_p(a), frame.tag(n), a.size, _p(mask), float(invalid)) == 0


def filter_field(frame, field, lower, upper, invalid=0, filtered_fields=None):
    src = frame.field(field)
    if src.shape != (frame.h, frame.w) or frame.tag(field) not in HANDLED:
        raise ValueError(SOURCE_MSG)
    names = _visited(frame, resolve_pixel_fields(frame, filtered_fields))
    check_invalid(frame, names, invalid)
    m = np.empty((frame.h, frame.w), np.uint8)
    assert lib().orc_fo_filter_mask(_p(m), _p(src), frame.tag(field), src.size, lower, upper) == 0
    _apply(frame, names, m, invalid)


def filter_uv(frame, coord_2d, lower, upper, invalid=0, filtered_fields=None, literal=True):
    """frame_ops::filter_uv with the C++ checks (frame_ops.cpp:240-253); literal=False masks "v" directly."""
    if coord_2d not in ("u", "v"):
        raise ValueError(f"coord_2d == {coord_2d} must be either 'u' or 'v'")
    size = frame.h if coord_2d == "u" else frame.w
    if lower > size or upper > size:
        raise ValueError(f"lower == {lower} and upper == {upper} must be in the range [0, {size}]")
    if lower > upper:
        raise ValueError(f"lower == {lower} must be less than upper == {upper}")
    names = resolve_pixel_fields(frame, filtered_fields)
    visited = _visited(frame, names)
    check_invalid(frame, visited, invalid)
    if coord_2d == "u":
        m = np.ones((frame.h, frame.w), np.uint8)
        m[lower:upper] = 0
        _apply(frame, visited, m, invalid)
        return
    for n in names:
        a = frame.field(n)
        if frame.tag(n) not in HANDLED:
            a[...] = 0          # destagger of a skipped type returns a zeroed field
            continue
        if literal:
            assert lib().orc_fo_uv_v_literal(_p(a), frame.tag(n), a.itemsize, _p(frame.shifts), frame.h, frame.w,
                                             lower, upper, float(invalid)) == 0
        else:
            m = np.empty((frame.h, frame.w), np.uint8)
            lib().orc_fo_uv_v_mask(_p(m), _p(frame.shifts), frame.h, frame.w, lower, upper)
            _apply(frame, [n], m, invalid)


def uv_v_mask(shifts, h, w, lower, upper):
    m = np.empty((h, w), np.uint8)
    lib().orc_fo_uv_v_mask(_p(m), _p(np.ascontiguousarray(shifts, np.int32)), h, w, lower, upper)
    return m


def mask(frame, fields, mask):
    mask = np.ascontiguousarray(mask, np.uint8)
    if mask.shape[0] != frame.h or mask.shape[1] != frame.w:
        raise ValueError("Used mask size doesn't match frame size")
    names = _visited(frame, resolve_pixel_fields(frame, list(fields) if fields else None))
    _apply(frame, names, mask, 0.0)


def xyz_mask(points, axis, lower, upper):
    """1 where the point's axis coordinate lies in [lower, upper], in the points' dtype."""
    pts = np.ascontiguousarray(points)
    n = pts.size // 3
    hit = np.empty(n, np.uint8)
    fn = lib().orc_fo_xyz_mask_f64 if pts.dtype == np.float64 else lib().orc_fo_xyz_mask_f32
    fn(_p(hit), _p(pts), n, axis, lower, upper)
    return hit


def filter_xyz(frame, points_of, axis_idx, lower=float("-inf"), upper=float("inf"), invalid=0,
               filtered_fields=None):
    """frame_ops.filter_xyz with points_of(range_field_name) -> (h, w, 3) points (projection and pose are the
    caller's: oracle.cartesian / oracle.dewarp)."""
    if axis_idx < 0 or axis_idx > 2:
        raise ValueError(f"axis_idx == {axis_idx} must be in the range [0, 2]")
    masks = {}
    for r, name in enumerate(("RANGE", "RANGE2")):
        if frame.has_field(name):
            masks[r] = xyz_mask(points_of(name), axis_idx, lower, upper).reshape(frame.h, frame.w)
    if not masks:
        return
    names = _visited(frame, resolve_pixel_fields(frame, filtered_fields, python=True))
    check_invalid(frame, names, invalid)
    for n in names:
        r = 1 if n in SECOND_RETURN else 0
        m = masks.get(r, masks.get(1 - r))
        a = frame.field(n)
        inv = np.array(float(invalid)).astype(a.dtype) if a.dtype.kind == "f" else np.array(int(np.trunc(invalid))).astype(a.dtype)
        a[m.astype(bool)] = inv


def select_rows(frame, indices):
    """select_by_index's pixel part: selected rows of every pixel field (any type, extra dims included); other
    fields copied (frame_ops.cpp:296-323)."""
    out = Frame(len(indices), frame.w, frame.shifts[np.asarray(indices)])
    for n in frame.fields:
        a, t, c = frame._f[n]
        out._f[n] = ((a[np.asarray(indices)].copy() if c == PIXEL_FIELD else a.copy()), t, c)
    out.body_to_world = frame.body_to_world.copy()
    out.headers = {k: np.copy(v) for k, v in frame.headers.items()}
    return out
