"""ctypes/numpy front-end of the image post-processing oracle (oracle/orc_image.c, built by oracle/image.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: restates AutoExposure, BeamUniformityCorrector and LocalToneMapper
(ouster_core/src/image_processing.cpp) with the same constructors and update(image, update_state) calls, on numpy
arrays updated in place.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libouster_oracle_image.so")
_SRCS = [os.path.join(_HERE, "orc_image.c"), os.path.join(_HERE, "orc_image_t.h")]


def build(force=False):
    """Compile the oracle (gcc); no-op when the .so is up to date."""
    if not force and os.path.exists(_LIB_PATH) and \
            all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in _SRCS):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "image.mk"])
    return _LIB_PATH


class State(C.Structure):
    """ob_image_state"""
    _fields_ = [("lo", C.c_double), ("hi", C.c_double), ("lo_state", C.c_double), ("hi_state", C.c_double),
                ("counter", C.c_int32), ("initialized", C.c_int32), ("dark_count_rows", C.c_uint32),
                ("reserved", C.c_uint32)]


class Params(C.Structure):
    """ob_image_params"""
    _fields_ = [("lo_percentile", C.c_double), ("hi_percentile", C.c_double), ("update_every", C.c_int32),
                ("color_correct", C.c_int32), ("damping", C.c_double), ("compress_dr_max_lum", C.c_double)]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        build()
    L = C.CDLL(_LIB_PATH)
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    for s in ("_f", "_d"):
        getattr(L, "orc_ae_update" + s).argtypes = [C.POINTER(State), C.POINTER(Params), vp, sz, sz, i32, i32]
        getattr(L, "orc_ltm_update" + s).argtypes = [C.POINTER(State), C.POINTER(Params), vp, sz, sz, i32]
        getattr(L, "orc_buc_update" + s).argtypes = [C.POINTER(State), vp, vp, sz, sz, i32]
        getattr(L, "orc_dark_count" + s).argtypes = [vp, sz, sz, vp]
        getattr(L, "orc_fullpivlu_fit" + s).argtypes = [vp, sz, vp]
        getattr(L, "orc_clahe_luts" + s).argtypes = [vp, i32, i32, vp]
    L.orc_f16_bits_fast.argtypes = [C.c_uint16]
    L.orc_f16_bits_fast.restype = C.c_uint32
    L.orc_f16_convert.argtypes = [vp, vp, sz]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _suffix(a):
    if a.dtype == np.float32:
        return "_f"
    if a.dtype == np.float64:
        return "_d"
    raise TypeError("float32 or float64 image expected")


def _check(a):
    if not (isinstance(a, np.ndarray) and a.flags["C_CONTIGUOUS"]):
        raise TypeError("a C-contiguous numpy array is expected")


def f16_to_f32(bits):
    """f16_bits_to_f32_bits_fast_nan_zero over an array of float16 (or uint16 bits): float32"""
    b = np.ascontiguousarray(np.asarray(bits).view(np.uint16))
    out = np.empty(b.shape, np.float32)
    lib().orc_f16_convert(_p(b), _p(out), b.size)
    return out


def fullpivlu_fit(rhs):
    """x = FullPivLU([1, i]).solve(rhs) in rhs's dtype"""
    rhs = np.ascontiguousarray(rhs)
    x = np.zeros(2, rhs.dtype)
    getattr(lib(), "orc_fullpivlu_fit" + _suffix(rhs))(_p(rhs), rhs.size, _p(x))
    return x


def dark_count(img):
    """compute_dark_count(img) in img's dtype"""
    img = np.ascontiguousarray(img)
    out = np.zeros(img.shape[0], img.dtype)
    getattr(lib(), "orc_dark_count" + _suffix(img))(_p(img), img.shape[0], img.shape[1], _p(out))
    return out


def clahe_luts(lum):
    """compute_clahe_luts(lum, 8, 8, 1024, 1.0): float32 [64, 1024]"""
    lum = np.ascontiguousarray(lum)
    out = np.zeros((64, 1024), np.float32)
    getattr(lib(), "orc_clahe_luts" + _suffix(lum))(_p(lum), lum.shape[0], lum.shape[1], _p(out))
    return out


class _Proc:
    def __init__(self, lo, hi, update_every, damping, compress=0.0, color_correct=False):
        self.params = Params(lo, hi, int(update_every), int(bool(color_correct)), damping, compress)
        self.st = State(-1.0, -1.0, -1.0, -1.0, 0, 0, 0, 0)

    def state(self):
        s = self.st
        return dict(lo=s.lo, hi=s.hi, lo_state=s.lo_state, hi_state=s.hi_state, counter=s.counter,
                    initialized=bool(s.initialized))


class AutoExposure(_Proc):
    def __init__(self, *args):
        if len(args) == 0:
            args = (0.1, 0.1, 3, 0.9)
        elif len(args) == 1:
            args = (0.1, 0.1, args[0], 0.9)
        elif len(args) == 3:
            args = tuple(args) + (0.9,)
        super().__init__(*args)

    def update(self, image, update_state=True):
        """mono (h, w) or rgb (h, w, 3) float32/float64 in place; float16 rgb returns a new float32 array"""
        if image.dtype == np.float16:
            out = f16_to_f32(image)
            self.update(out, update_state)
            return out
        _check(image)
        rgb = image.ndim == 3
        getattr(lib(), "orc_ae_update" + _suffix(image))(C.byref(self.st), C.byref(self.params), _p(image),
                                                         image.shape[0], image.shape[1], int(rgb),
                                                         int(bool(update_state)))
        return None


class LocalToneMapper(_Proc):
    def __init__(self, lo=0.0, hi=0.2, update_every=1, damping=0.3, compress_dr_max_lum=0.2, color_correct=True):
        if isinstance(compress_dr_max_lum, bool):
            compress_dr_max_lum = 0.2 if compress_dr_max_lum else 0.0
        super().__init__(lo, hi, update_every, damping, compress_dr_max_lum, color_correct)

    def update(self, image, update_state=True):
        if image.dtype == np.float16:
            out = f16_to_f32(image)
            self.update(out, update_state)
            return out
        _check(image)
        getattr(lib(), "orc_ltm_update" + _suffix(image))(C.byref(self.st), C.byref(self.params), _p(image),
                                                          image.shape[0], image.shape[1], int(bool(update_state)))
        return None


class BeamUniformityCorrector:
    def __init__(self):
        self.st = State(-1.0, -1.0, -1.0, -1.0, 0, 0, 0, 0)
        self.dark = np.zeros(0)

    def update(self, image, update_state=True):
        _check(image)
        h = image.shape[0]
        if self.dark.size != h:
            self.dark = np.zeros(h)
        getattr(lib(), "orc_buc_update" + _suffix(image))(C.byref(self.st), _p(self.dark), _p(image), h,
                                                          image.shape[1], int(bool(update_state)))

    def state(self):
        return dict(counter=self.st.counter, dark_count=self.dark[:self.st.dark_count_rows].copy())
