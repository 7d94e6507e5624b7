"""ctypes/numpy front-end of the pose-interpolation oracle (oracle/orc_pose.c, built by oracle/pose.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates core::interp_pose in both forms
(ouster_core/include/ouster/core/pose_util.h:194-434), PoseH::log / PoseV::exp and the constant-velocity deskew of a
frame set (ouster_mapping/src/deskew_method.cpp:29-71, slam_util.cpp:129-140).  Errors raise ValueError with the
reference's texts (std::invalid_argument).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_pose.so")
_SRCS = [os.path.join(_HERE, "orc_pose.c"), os.path.join(_HERE, "orc_align.c")]

OK, KNOT_ORDER, ZERO_DURATION, DESCENT = range(4)


def build(force=False):
    """Compile the oracle (gcc); no-op when the .so is up to date."""
    if (not force and os.path.exists(_LIB_PATH)
            and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in _SRCS)):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "pose.mk"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    build()
    L = C.CDLL(_LIB_PATH)
    vp, sz, i32, d = C.c_void_p, C.c_size_t, C.c_int, C.c_double
    L.orc_poseh_log.argtypes = [vp, vp]
    L.orc_posev_exp.argtypes = [vp, vp]
    L.orc_inverse4.argtypes = [vp, vp]
    L.orc_interp_pose.argtypes = [vp, sz, vp, sz, i32, vp, i32, vp, vp]
    L.orc_interp_pose.restype = i32
    L.orc_frames_interp_pose.argtypes = [vp, vp, vp, vp, sz, d, vp, d, vp, vp]
    L.orc_frames_interp_pose.restype = i32
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _fmt(bits, is_int):
    """std::to_string of the value whose 8 bytes are `bits`."""
    b = np.array([bits], np.int64)
    return str(int(b[0])) if is_int else "%f" % float(b.view(np.float64)[0])


def message(err, is_int=False):
    """The reference's text for the error words (kind, index, frame, value bits of x[index], x[index - 1])."""
    kind = int(err[0])
    if kind == KNOT_ORDER:
        return "input x_known values are not monotonically increasing or values repeated"
    if kind == ZERO_DURATION:
        return "Cannot interpolate with zero duration between poses"
    if kind == DESCENT:
        return ("x_interp values must be monotonically increasing: " + _fmt(err[3], is_int) + " < "
                + _fmt(err[4], is_int))
    return None


def poseh_log(m):
    m = np.ascontiguousarray(m, np.float64).reshape(4, 4)
    v = np.empty(6)
    lib().orc_poseh_log(_ptr(m), _ptr(v))
    return v


def posev_exp(v):
    v = np.ascontiguousarray(v, np.float64).reshape(6)
    m = np.empty((4, 4))
    lib().orc_posev_exp(_ptr(v), _ptr(m))
    return m


def inverse4(m):
    m = np.ascontiguousarray(m, np.float64).reshape(4, 4)
    r = np.empty((4, 4))
    lib().orc_inverse4(_ptr(m), _ptr(r))
    return r


def interp_pose_words(x_interp, x_known, poses_known, two_pose=False):
    """-> (n x 4 x 4 float64 or None on error, error words).  x as float64 or int64 (the dtype of x_interp)."""
    is_int = np.asarray(x_interp).dtype.kind in "iu"
    dt = np.int64 if is_int else np.float64
    x = np.ascontiguousarray(x_interp, dt).reshape(-1)
    k = np.ascontiguousarray(x_known, dt).reshape(-1)
    pk = np.ascontiguousarray(poses_known, np.float64).reshape(-1, 16)
    if len(k) != len(pk):
        raise ValueError("x_known and poses_known sizes are not matching")
    if not two_pose and len(k) < 2:
        raise ValueError("Not enough evaluation poses for interpolation")
    out = np.empty((max(len(x), 1), 4, 4))
    err = np.zeros(5, np.int64)
    kind = lib().orc_interp_pose(_ptr(x), len(x), _ptr(k), len(k), 1 if is_int else 0, _ptr(pk), int(two_pose),
                                 _ptr(out), _ptr(err))
    return (out[:len(x)] if kind == OK else None), err


def interp_pose(x_interp, x_known, poses_known):
    """core::interp_pose(x_interp, x_known, poses_known): n x 4 x 4 float64, ValueError with the reference's text."""
    out, err = interp_pose_words(x_interp, x_known, poses_known)
    if out is None:
        raise ValueError(message(err, np.asarray(x_interp).dtype.kind in "iu"))
    return out


def interp_pose_two(x_interp, t0, x0, t1, x1):
    """core::interp_pose(x_interp, t0, x0, t1, x1)."""
    dt = np.asarray(x_interp).dtype
    out, err = interp_pose_words(x_interp, np.array([t0, t1], dt), np.stack([x0, x1]), two_pose=True)
    if out is None:
        raise ValueError(message(err, dt.kind in "iu"))
    return out


def interp_pose_float(x_interp, x_known, poses_known):
    """interp_pose_float: float32 known poses widened, each result rounded once to float32."""
    return interp_pose(x_interp, x_known, np.asarray(poses_known, np.float32).astype(np.float64)).astype(np.float32)


def frames_interp_pose(frames, t0, x0, t1=None, x1=None):
    """ConstantVelocityDeskewMethod::update on a list of (timestamps, status, poses w x 4 x 4 float64) or None,
    poses updated in place; x1 None: init_valid_column_poses(x0).  -> error words (kind 0 on success)."""
    n = len(frames)
    ts = (C.c_void_p * n)()
    stv = (C.c_void_p * n)()
    pv = (C.c_void_p * n)()
    w = (C.c_size_t * n)()
    keep = []
    for i, f in enumerate(frames):
        if f is None:
            continue
        t, s, p = f
        t = np.ascontiguousarray(t, np.uint64)
        s = np.ascontiguousarray(s, np.uint32)
        assert p.dtype == np.float64 and p.flags.c_contiguous
        keep += [t, s]
        ts[i], stv[i], pv[i], w[i] = t.ctypes.data, s.ctypes.data, p.ctypes.data, len(t)
    a0 = np.ascontiguousarray(x0, np.float64).reshape(16)
    a1 = None if x1 is None else np.ascontiguousarray(x1, np.float64).reshape(16)
    err = np.zeros(5, np.int64)
    lib().orc_frames_interp_pose(C.cast(ts, C.c_void_p), C.cast(stv, C.c_void_p), C.cast(pv, C.c_void_p),
                                 C.cast(w, C.c_void_p), n, float(t0), _ptr(a0), float(t1 or 0.0),
                                 None if a1 is None else _ptr(a1), _ptr(err))
    return err
