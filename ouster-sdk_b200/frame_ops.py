"""Frame operations on the GPU (DESIGN f-10): the functions of `ouster.sdk.core.frame_ops`
(python/src/ouster/sdk/core/frame_ops.py, bound from ouster_core/src/frame_ops.cpp) with the same names, keyword
defaults and ValueError texts.

Each takes a host `LidarFrame`, a `pyapi.DeviceLidarScan`, or a list of frames of one shape, which then go to the
GPU in one launch.  A `DeviceLidarScan` is modified in place on its CUDA tensors, on the torch stream, and nothing
waits for the host; `select_by_index` / `reduce_by_factor` of one return a new `DeviceLidarScan`.  Host frames are
staged through the C library and are final when the call returns.

    from ouster_sdk_b200 import frame_ops
    frame_ops.clip(scan, ["RANGE"], 500, 20000)
    frame_ops.filter_xyz(scan, pyapi.XYZLutFloat(info), 2, -0.5, 0.5)
    small = frame_ops.reduce_by_factor(scan, 2, update_metadata=True)

Semantics follow the reference's code (DESIGN §9 lists where it is undefined and what happens here instead):
comparisons in double, `invalid` cast to each field's type, FLOAT16 and the other non-numeric types skipped,
`filter_uv("v")` on destaggered columns with its zero-fill of skipped types, the second-return mask for RANGE2,
SIGNAL2, REFLECTIVITY2 and FLAGS2 in `filter_xyz`.  Every argument is checked before the launch, so a call that
raises modifies nothing.
"""
import ctypes as C
import re

import numpy as np

from . import _capi
from . import core as _c
from .host import TAG_NP, LidarFrame, SensorInfo

PIXEL_FIELD = 1
_HANDLED = set(range(1, 11))        # u8..u64, i8..i64, f32, f64 (impl::visit_field_2d)
_SECOND_RETURN = {"RANGE2", "SIGNAL2", "REFLECTIVITY2", "FLAGS2"}
_DIMS_MSG = ("Field: Eigen array conversion failed due to dimension mismatch. Underlying data has {} dimensions "
             "but must have 2 dimensions.")
_SOURCE_MSG = "filter_field requires a pixel field with shape (h, w) to build a mask"


# ---- frames ------------------------------------------------------------------------------------------------------
class _Frame:
    """One frame's pixel fields as (pointer, tag, shape), whether host arrays or CUDA tensors."""

    def __init__(self, frame):
        self.frame = frame
        self.device = hasattr(frame, "host") and hasattr(frame, "_fields")   # pyapi.DeviceLidarScan
        self.host = frame.host if self.device else frame
        self.h, self.w = frame.h, frame.w
        self.names = list(frame.fields)

    def tag(self, name):
        return self.host.field_tag(name)

    def field_class(self, name):
        return self.host.field_class(name)

    def array(self, name):
        return self.frame.field(name)

    def ptr(self, name):
        return _c._ptr(self.array(name))

    def shape(self, name):
        return tuple(self.array(name).shape)

    @property
    def sensor_info(self):
        return getattr(self.frame, "sensor_info", None) if not self.device else self.frame.info


def _frames(frame):
    many = isinstance(frame, (list, tuple))
    fs = [_Frame(f) for f in (frame if many else [frame])]
    if fs:
        kinds = {f.device for f in fs}
        shapes = {(f.h, f.w) for f in fs}
        if len(kinds) > 1 or len(shapes) > 1:
            raise ValueError("frames of one call must share their shape and their memory kind")
    return fs


def _resolve_pixel_fields(fr, filtered_fields, python=False):
    """resolve_pixel_fields (frame_ops.cpp:19-62) / _resolve_pixel_fields (frame_ops.py:17-39): missing names are
    ignored, non-pixel names in an explicit list raise (the binding's text, or the Python module's with `python`)."""
    requested = list(filtered_fields) if filtered_fields is not None else fr.names
    present = [f for f in requested if f in fr.names]
    non_pixel = [f for f in present if fr.field_class(f) != PIXEL_FIELD]
    if filtered_fields is not None and non_pixel:
        if python:
            raise ValueError(f"Only PIXEL_FIELD frame fields are supported here; requested non-pixel fields: "
                             f"{non_pixel}")
        raise ValueError("Only PIXEL_FIELD frame fields are supported here; requested non-pixel fields: ["
                         + ", ".join(non_pixel) + "]")
    return [f for f in present if fr.field_class(f) == PIXEL_FIELD]


def _targets(fr, names, role_of=None):
    """(name, tag, role) of the fields the per-type visit writes; raises the reference's dimension text for a
    handled type that is not (h, w)."""
    out = []
    for name in names:
        tag = fr.tag(name)
        if tag not in _HANDLED:
            continue
        shape = fr.shape(name)
        if len(shape) != 2:
            raise ValueError(_DIMS_MSG.format(len(shape)))
        out.append((name, tag, role_of(name) if role_of else _capi.OB_FRAME_TARGET))
    return out


def _run(fs, predicate, per_frame, lower=0.0, upper=0.0, invalid=0.0, shifts=None, lut=None, poses=None, axis=0,
         keep=()):
    """One ob_frame_mask_fields call; per_frame[i] lists (pointer, tag, role, elem_bytes) of frame i."""
    ents = [(p, t, r, i, eb) for i, lst in enumerate(per_frame) for (p, t, r, eb) in lst]
    if not fs or not ents:
        return
    tab = (_capi.FrameField * len(ents))()
    for k, (p, t, r, i, eb) in enumerate(ents):
        tab[k].data, tab[k].type, tab[k].role, tab[k].frame, tab[k].elem_bytes = p, t, r, i, eb
    io = _capi.FrameOpsIO()
    io.n_frames, io.h, io.w, io.predicate = len(fs), fs[0].h, fs[0].w, predicate
    io.fields, io.n_fields = tab, len(ents)
    io.lower, io.upper, io.invalid = float(lower), float(upper), float(invalid)
    sh = None
    if shifts is not None:
        sh = np.ascontiguousarray(shifts, np.int32)
        io.pixel_shift_by_row = sh.ctypes.data_as(C.POINTER(C.c_int32))
    io.lut = lut._h if lut is not None else None
    io.poses = _c._ptr(poses) if poses is not None else None
    io.axis = int(axis)
    st = _c._stream_for(fs[0].array(fs[0].names[0]) if fs[0].device else None)
    _c.check(_c.lib.ob_frame_mask_fields(C.byref(io), st.h))
    if fs[0].device:
        _keep(fs[0], (tab, sh, poses) + tuple(keep))


def _keep(fr, objs):
    """Device calls return before the GPU reads their inputs: hold host-side inputs until the next call."""
    fr.frame._frame_ops_keep = objs


def _invalid_number(invalid):
    try:
        return float(invalid)
    except (TypeError, OverflowError) as e:
        raise ValueError(str(e)) from None


# ---- operations on pixel values --------------------------------------------------------------------------------
def clip(frame, fields, lower, upper, invalid=0):
    """frame_ops::clip (frame_ops.cpp:151-163, 211-218): a value is kept iff lower <= (double)v <= upper, else it
    becomes static_cast<T>(invalid); NaN values become invalid.  `fields` empty: every pixel field."""
    fs = _frames(frame)
    invalid = _invalid_number(invalid)
    per = []
    for fr in fs:
        names = _resolve_pixel_fields(fr, list(fields) if fields else None)
        per.append([(fr.ptr(n), t, r, 0) for n, t, r in _targets(fr, names)])
    _run(fs, _capi.OB_FRAME_CLIP, per, lower, upper, invalid)


def filter_field(frame, field, lower, upper, invalid=0, filtered_fields=None):
    """frame_ops::filter_field (frame_ops.cpp:165-183, 220-236): pixels whose `field` value lies inside
    [lower, upper] become invalid in every target (the code's meaning; a NaN source pixel is kept).  The mask is
    taken from the source's values before any write, so the source may be a target."""
    fs = _frames(frame)
    invalid = _invalid_number(invalid)
    per = []
    for fr in fs:
        if field not in fr.names:
            raise IndexError(f"Field '{field}' not found in LidarFrame.")
        if fr.shape(field) != (fr.h, fr.w) or fr.tag(field) not in _HANDLED:
            raise ValueError(_SOURCE_MSG)
        lst = [(fr.ptr(n), t, r, 0) for n, t, r in _targets(fr, _resolve_pixel_fields(fr, filtered_fields))]
        lst.append((fr.ptr(field), fr.tag(field), _capi.OB_FRAME_SOURCE, 0))
        per.append(lst)
    _run(fs, _capi.OB_FRAME_VALUE, per, lower, upper, invalid)


def filter_uv(frame, coord_2d, lower, upper, invalid=0, filtered_fields=None):
    """frame_ops.filter_uv (frame_ops.py:42-81, frame_ops.cpp:238-276): "u" invalidates rows [lower, upper), "v"
    destaggered columns [lower, upper).  Floats in [0, 1] are fractions of the axis, -inf / inf its edges.  "v"
    also zero-fills every pixel field of a type the per-type visit skips, as the reference's destagger does."""
    fs = _frames(frame)
    if coord_2d not in ['u', 'v']:
        raise ValueError(f"coord_2d == {coord_2d} must be either 'u' or 'v'")
    if not fs:
        return
    coord_size = fs[0].h if coord_2d == 'u' else fs[0].w

    def _interpret_as_int(val):
        if val == float("-inf"):
            return 0
        if val == float("inf"):
            return coord_size
        if 0 <= val <= 1:
            return int(coord_size * val)
        return int(val)

    if isinstance(lower, float):
        lower = _interpret_as_int(lower)
    if isinstance(upper, float):
        upper = _interpret_as_int(upper)
    if lower < 0 or upper > coord_size:
        raise ValueError(f"lower == {lower} and upper == {upper} must be in the range [0, {coord_size}]")
    if lower > upper:
        raise ValueError(f"lower == {lower} must be less than upper == {upper}")
    invalid = _invalid_number(invalid)
    per = []
    shifts = None
    for fr in fs:
        names = _resolve_pixel_fields(fr, filtered_fields)
        lst = [(fr.ptr(n), t, r, 0) for n, t, r in _targets(fr, names)]
        if coord_2d == 'v':
            info = fr.sensor_info
            if info is None:
                raise ValueError("filter_uv 'v' requires frame.sensor_info")
            sh = np.asarray(info.pixel_shift_by_row, np.int32)
            if shifts is None:
                shifts = sh
            elif not np.array_equal(sh, shifts):
                # one launch takes one shift table: frames that stagger differently go to separate calls
                raise ValueError("frames of one filter_uv('v') call must share pixel_shift_by_row")
            for n in names:
                if fr.tag(n) in _HANDLED:
                    continue
                a = fr.array(n)   # a type the per-type visit skips: destagger() hands back a zeroed field
                eb = (a.numel() * a.element_size() if hasattr(a, "numel") else a.nbytes) // (fr.h * fr.w)
                if eb:
                    lst.append((fr.ptr(n), fr.tag(n), _capi.OB_FRAME_ZERO, eb))
        per.append(lst)
    if coord_2d == 'u':
        _run(fs, _capi.OB_FRAME_ROWS, per, lower, upper, invalid)
    else:
        _run(fs, _capi.OB_FRAME_COLS, per, lower, upper, invalid, shifts=shifts)


def mask(frame, fields, mask):
    """frame_ops.mask (frame_ops.py:139-150, frame_ops.cpp:185-199, 278-286): pixels whose mask byte is 0 become
    0 in the fields (empty: every pixel field).  `mask` may be a numpy array or a CUDA tensor."""
    fs = _frames(frame)
    if not fs:
        return
    h, w = fs[0].h, fs[0].w
    if mask.shape[0] != h or mask.shape[1] != w:
        raise ValueError(f"Used mask size {tuple(mask.shape)} doesn't match frame size"
                         " ({frame.h}, {frame.w}")
    if len(mask.shape) != 2:
        raise ValueError("Used mask size doesn't match frame size")
    if _c._is_torch(mask):
        import torch
        m = mask.to(torch.uint8).contiguous() if mask.dtype != torch.uint8 else mask.contiguous()
        if fs[0].device and not m.is_cuda:
            m = m.to(fs[0].array(fs[0].names[0]).device)
    else:
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        if fs[0].device:
            import torch
            m = torch.as_tensor(m, device=fs[0].array(fs[0].names[0]).device)
    per = []
    for fr in fs:
        names = _resolve_pixel_fields(fr, list(fields) if fields else None)
        lst = [(fr.ptr(n), t, r, 0) for n, t, r in _targets(fr, names)]
        lst.append((_c._ptr(m), 1, _capi.OB_FRAME_SOURCE, 0))
        per.append(lst)
    _run(fs, _capi.OB_FRAME_VALUE, per, 0.0, 0.0, 0.0, keep=(m,))


def filter_xyz(frame, xyzlut, axis_idx, lower=float("-inf"), upper=float("inf"), invalid=0, filtered_fields=None,
               dewarp_points=False):
    """frame_ops.filter_xyz (frame_ops.py:83-136): pixels whose point lies inside [lower, upper] on `axis_idx`
    become invalid.  RANGE2, SIGNAL2, REFLECTIVITY2 and FLAGS2 take the second return's mask, the other fields the
    first's; each falls back to the other when its own is absent.

    `xyzlut` a `pyapi.XYZLut` / `XYZLutFloat` (or `XYZLutT`): the projection (and, with `dewarp_points`, each
    column's `body_to_world` pose) is fused into the launch, in the LUT's dtype.  Any other callable is called on
    the range field and its (h, w, 3) result is the predicate's input, compared in its own dtype."""
    if axis_idx < 0 or axis_idx > 2:
        raise ValueError(f"axis_idx == {axis_idx} must be in the range [0, 2]")
    fs = _frames(frame)
    invalid = _invalid_number(invalid)
    lut = getattr(xyzlut, "_lut", xyzlut) if isinstance(getattr(xyzlut, "_lut", xyzlut), _c.XYZLutT) else None
    per, keep, poses = [], [], None
    fused = lut is not None
    for fr in fs:
        srcs = {}
        for r, name in enumerate(("RANGE", "RANGE2")):
            if name not in fr.names:
                continue
            if fused:
                if fr.shape(name) != (lut.h, lut.w):
                    raise ValueError("Frame dimensions do not match lut.")
                srcs[r] = (fr.ptr(name), 3)
            else:
                pts = xyzlut(fr.array(name))
                if dewarp_points:
                    from . import pyapi
                    pts = pyapi.dewarp(pts, fr.host.body_to_world)
                pts = _points(pts, fr)
                keep.append(pts)
                srcs[r] = (_c._ptr(pts), 10 if str(pts.dtype).endswith("float64") else 9)
        if not srcs:
            per.append([])
            continue

        def role_of(name, srcs=srcs):
            second = name in _SECOND_RETURN
            if second:
                return _capi.OB_FRAME_TARGET2 if 1 in srcs else _capi.OB_FRAME_TARGET
            return _capi.OB_FRAME_TARGET if 0 in srcs else _capi.OB_FRAME_TARGET2

        lst = [(fr.ptr(n), t, r, 0)
               for n, t, r in _targets(fr, _resolve_pixel_fields(fr, filtered_fields, python=True), role_of)]
        for r, (p, t) in srcs.items():
            lst.append((p, t, _capi.OB_FRAME_SOURCE if r == 0 else _capi.OB_FRAME_SOURCE2, 0))
        per.append(lst)
    if fused:
        if dewarp_points:
            dt = lut.dtype
            poses = np.ascontiguousarray(np.stack([fr.host.body_to_world for fr in fs]), dt)
            if fs and fs[0].device:
                import torch
                poses = torch.as_tensor(poses, device=fs[0].array(fs[0].names[0]).device)
        _run(fs, _capi.OB_FRAME_XYZ_RANGE, per, lower, upper, invalid, lut=lut, poses=poses, axis=axis_idx,
             keep=(lut,))
    else:
        _run(fs, _capi.OB_FRAME_XYZ_POINTS, per, lower, upper, invalid, axis=axis_idx, keep=tuple(keep))


def _points(pts, fr):
    """(h, w, 3) float32 / float64 points of a callable LUT, as a contiguous array of the frame's memory kind."""
    if _c._is_torch(pts):
        import torch
        if pts.dtype not in (torch.float32, torch.float64):
            pts = pts.double()
        if fr.device and not pts.is_cuda:
            pts = pts.to(fr.array(fr.names[0]).device)
        if not fr.device and pts.is_cuda:
            raise ValueError("points of a host frame must be host arrays")
        pts = pts.contiguous()
    else:
        pts = np.asarray(pts)
        if pts.dtype not in (np.float32, np.float64):
            pts = pts.astype(np.float64)
        pts = np.ascontiguousarray(pts)
        if fr.device:
            import torch
            pts = torch.as_tensor(pts, device=fr.array(fr.names[0]).device)
    if tuple(pts.shape)[-1] != 3 or int(np.prod(tuple(pts.shape))) != fr.h * fr.w * 3:
        raise ValueError("xyzlut must return (h, w, 3) points")
    return pts


# ---- row selection -------------------------------------------------------------------------------------------
def _validate_beam_indices(indices, height):
    if not indices:
        raise ValueError("beam indices can't be empty")
    if len(indices) != len(set(indices)):
        raise ValueError("beam indices can't contain duplicates")
    invalid_indices = [i for i in indices if i < 0 or i >= height]
    if invalid_indices:
        raise ValueError(f"beam indices {invalid_indices} must be in the range [0, {height})")


def _reduce_factor_to_slice(factor, height):
    if factor == height:
        return slice(height // 2, height // 2 + 1, None)
    return slice(None, None, factor)


def _reduce_factor_to_indices(factor, height):
    if factor <= 0:
        raise ValueError(f"factor == {factor} can't be negative")
    if not (height / factor).is_integer():
        raise ValueError(f"factor == {factor} must be a divisor of {height}")
    return list(range(height))[_reduce_factor_to_slice(factor, height)]


_PRODUCT_RE = re.compile(r"^(\w+)-(\d+|DOME)?(?:-(MAX))?(?:-(\d+))?(?:-(RGB))?(?:-((?!SR)\w+))?-?(SR)?", re.ASCII)


def product_info(prod_line):
    """ProductInfo::create_product_info (sensor_info.cpp:442-470) -> dict of its members."""
    if not prod_line:
        return {"full_product_info": "", "form_factor": "", "short_range": False, "beam_config": "",
                "beam_count": 0, "rgb": False}
    m = _PRODUCT_RE.search(prod_line)
    if m is None:
        raise RuntimeError(f'Product Info "{prod_line}" is not a recognized product info')
    g = [m.group(i) or "" for i in range(8)]
    try:
        beam_count = int(g[4])
    except ValueError:
        beam_count = 0
    return {"full_product_info": prod_line, "form_factor": g[1] + g[2] + g[3], "short_range": bool(g[7]),
            "beam_config": g[6] or "U", "beam_count": beam_count, "rgb": g[5] == "RGB"}


def form_factor_prod_line(prod_line, v_res):
    """form_factor_prod_line (frame_ops.cpp:110-124): the product line of a sensor with v_res beams."""
    pi = product_info(prod_line)
    ff = pi["form_factor"]
    if "MAX" in ff:
        ff = "OS" + ff[2:3] + "MAX"
    elif ff and ff[-1].isdigit():
        ff = ff[:-1] + "-" + ff[-1]
    ff = ff + "-" + str(v_res)
    if pi["rgb"]:
        ff += "-RGB"
    return ff


def select_by_index_metadata(metadata, indices):
    """frame_ops::select_by_index_metadata (frame_ops.cpp:339-362): a new SensorInfo of len(indices) rows with the
    selected shifts and beam angles and the rewritten product line (SensorInfo here has no zone_set)."""
    indices = [int(i) for i in indices]
    _validate_beam_indices(indices, metadata.h)
    idx = np.asarray(indices, np.int64)
    out = SensorInfo(metadata.profile, len(indices), metadata.w, metadata.columns_per_packet,
                     metadata.header_type, np.asarray(metadata.pixel_shift_by_row)[idx], metadata.init_id,
                     metadata.sn, metadata.fw_rev, metadata.column_window,
                     prod_line=form_factor_prod_line(metadata.prod_line, len(indices)))
    if getattr(metadata, "beam_azimuth_angles", None) is not None:
        out.set_intrinsics(np.asarray(metadata.beam_azimuth_angles)[idx],
                           np.asarray(metadata.beam_altitude_angles)[idx], metadata.beam_to_lidar_transform,
                           metadata.lidar_to_sensor_transform, getattr(metadata, "sensor_to_body", None))
    return out


def reduce_by_factor_metadata(metadata, factor):
    return select_by_index_metadata(metadata, _reduce_factor_to_indices(factor, metadata.h))


def _gather(pairs, rows, src_rows):
    """One ob_frame_select_rows call over (src, dst) arrays of the same row length."""
    if not pairs:
        return
    tab = (_capi.FrameRowsEntry * len(pairs))()
    for k, (s, d) in enumerate(pairs):
        nb = int(np.prod(tuple(s.shape)[1:])) * _c._itemsize(s)
        tab[k].src, tab[k].dst, tab[k].row_bytes, tab[k].src_rows = _c._ptr(s), _c._ptr(d), nb, src_rows
    r = np.asarray(rows, np.uint32)
    io = _capi.FrameRowsIO()
    io.entries, io.n_entries, io.n_rows = tab, len(pairs), len(rows)
    io.rows = r.ctypes.data_as(C.POINTER(C.c_uint32))
    _c.check(_c.lib.ob_frame_select_rows(C.byref(io), _c._stream_for(pairs[0][0]).h))


def select_by_index(frame, indices, update_metadata=False):
    """frame_ops::select_by_index (frame_ops.cpp:296-330): a new frame of the selected rows of every pixel field
    (extra dims included); headers, frame_id, status, countdowns and body_to_world are copied.  The result's
    sensor_info is None unless `update_metadata`, as in the reference.  A list of frames gives a list, gathered in
    one launch."""
    many = isinstance(frame, (list, tuple))
    fs = _frames(frame)
    indices = [int(i) for i in indices]
    for fr in fs:
        _validate_beam_indices(indices, fr.h)
        if fr.sensor_info is None:
            raise ValueError("select_by_index requires frame.sensor_info")
    outs, pairs, metas = [], [], {}
    for fr in fs:
        key = id(fr.sensor_info)
        if key not in metas:   # frames of one sensor share the selected metadata
            metas[key] = select_by_index_metadata(fr.sensor_info, indices)
        info = metas[key]
        if fr.device:
            from . import pyapi
            dev = fr.array(fr.names[0]).device
            out = pyapi.DeviceLidarScan(info, dev.index)
            _copy_headers(fr.host, out.host)
            for n in list(out._fields):
                if n not in fr.names:
                    del out._fields[n]
            for n in fr.names:
                s = fr.array(n)
                cls = fr.field_class(n)
                if n not in out.host.fields:
                    out.host.add_field(n, TAG_NP.get(fr.tag(n), np.uint8), _extra(fr.shape(n), cls), tag=fr.tag(n),
                                       field_class=cls)
                if cls != PIXEL_FIELD:
                    out._fields[n] = s.clone()   # non-pixel fields are copied unchanged
                    continue
                if n not in out._fields or tuple(out._fields[n].shape[1:]) != tuple(s.shape[1:]):
                    import torch
                    out._fields[n] = torch.empty((len(indices),) + tuple(s.shape[1:]), dtype=s.dtype, device=dev)
                pairs.append((s.contiguous(), out._fields[n]))
            if not update_metadata:
                out.info = None
        else:
            out = LidarFrame(info)
            _copy_headers(fr.host, out)
            for n in fr.names:
                cls = fr.field_class(n)
                if n not in out.fields:
                    out.add_field(n, TAG_NP.get(fr.tag(n), np.uint8), _extra(fr.shape(n), cls), tag=fr.tag(n),
                                  field_class=cls)
                if cls != PIXEL_FIELD:
                    out.field(n)[...] = fr.array(n)   # non-pixel fields are copied unchanged
                    continue
                pairs.append((np.ascontiguousarray(fr.array(n)), out.field(n)))
            out.sensor_info = info if update_metadata else None
        outs.append(out)
    _gather(pairs, indices, fs[0].h if fs else 0)
    return outs if many else outs[0]


def _extra(shape, field_class):
    """the extra dimension of a field of this shape and class (LidarFrame::add_field's extra_dims)"""
    lead = {PIXEL_FIELD: 2, 2: 1, 3: 1}.get(field_class, 0)
    return int(np.prod(shape[lead:])) if len(shape) > lead else 1


def _copy_headers(src, dst):
    """the headers select_by_index copies (frame_ops.cpp:302-311); alert_flags are not among them"""
    dst.timestamp[:] = src.timestamp
    dst.measurement_id[:] = src.measurement_id
    dst.status[:] = src.status
    dst.packet_timestamp[:] = src.packet_timestamp
    dst.body_to_world[:] = src.body_to_world
    dst.frame_id = src.frame_id
    dst.set_status(*src.status_tuple())


def reduce_by_factor(frame, factor, update_metadata=False):
    """frame_ops::reduce_by_factor: select_by_index on every factor-th row (the middle row when factor == h)."""
    fs = _frames(frame)
    h = fs[0].h if fs else 0
    return select_by_index(frame, _reduce_factor_to_indices(factor, h), update_metadata)


def reduce_factor_to_indices(factor, height):
    return _reduce_factor_to_indices(factor, height)
