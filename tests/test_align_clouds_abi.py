"""CPU-side checks of ob_align_clouds (DESIGN f-14): struct sizes, the reference's error texts in its order (checked
before the device is touched) and OB_NO_DEVICE without a GPU."""
import ctypes

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import align_clouds as oac

ob = graft.load_package()
capi = ob._capi
lib = capi.lib


def test_structs_in_abi_sizeof_match_ctypes():
    for name, cls in {"ob_align_clouds_trace": capi.AlignCloudsTrace, "ob_align_clouds_io": capi.AlignCloudsIO}.items():
        assert lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name
    # the oracle fills the same trace layout
    assert ctypes.sizeof(oac.Trace) == ctypes.sizeof(capi.AlignCloudsTrace)
    assert [f[0] for f in oac.Trace._fields_] == [f[0] for f in capi.AlignCloudsTrace._fields_]


def _io(s_cols=3, t_cols=3, sn=None, tn=None, n=5):
    pts = np.zeros((n, 3))
    pose = np.zeros((4, 4))
    io = capi.AlignCloudsIO()
    for rows in (io.source, io.target):
        rows.dtype, rows.points, rows.n = capi.OB_F64, pts.ctypes.data, n
    io.source_cols, io.target_cols = s_cols, t_cols
    if sn is not None:
        io.source_normals, io.source_normal_rows, io.source_normal_cols = pts.ctypes.data, sn[0], sn[1]
    if tn is not None:
        io.target_normals, io.target_normal_rows, io.target_normal_cols = pts.ctypes.data, tn[0], tn[1]
    io.pose = pose.ctypes.data
    return io, (pts, pose)


@pytest.mark.parametrize("kw,text", [
    (dict(s_cols=4, t_cols=2), "source_points must have shape (N, 3)"),
    (dict(sn=(5, 2), tn=(4, 3)), "source_normals must have shape (N, 3)"),
    (dict(sn=(4, 3), t_cols=4), "source_points and source_normals must have the same number of rows"),
    (dict(sn=(5, 3), t_cols=4), "target_points must have shape (N, 3)"),
    (dict(sn=(5, 3), tn=(5, 4)), "target_normals must have shape (N, 3)"),
    (dict(sn=(5, 3), tn=(6, 3)), "target_points and target_normals must have the same number of rows"),
    (dict(sn=(5, 3)), "source_normals and target_normals must both be given or both be omitted"),
    (dict(tn=(5, 3)), "source_normals and target_normals must both be given or both be omitted"),
])
def test_error_texts_in_order(kw, text):
    io, keep = _io(**kw)
    assert lib.ob_align_clouds(ctypes.byref(io), None) == capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error().decode() == text
    with pytest.raises(ValueError, match="^" + text.replace("(", r"\(").replace(")", r"\)") + "$"):
        n = 5
        sp = np.zeros((n, kw.get("s_cols", 3)))
        tp = np.zeros((n, kw.get("t_cols", 3)))
        sn = None if "sn" not in kw else np.zeros((kw["sn"][0], kw["sn"][1]))
        tn = None if "tn" not in kw else np.zeros((kw["tn"][0], kw["tn"][1]))
        ob.core.align_clouds(sp, tp, sn, tn)


def test_no_device():
    io, keep = _io(sn=(5, 3), tn=(5, 3))
    rc = lib.ob_align_clouds(ctypes.byref(io), None)
    if ob.core.device_count() == 0:
        assert rc == capi.OB_NO_DEVICE
        with pytest.raises(Exception, match="no CUDA device"):
            ob.core.align_clouds(np.zeros((5, 3)), np.zeros((5, 3)))
    else:
        assert rc == capi.OB_INVALID_ARGUMENT and lib.ob_last_error() == b"null pointer"
