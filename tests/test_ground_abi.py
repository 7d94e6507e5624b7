"""CPU-side checks of ob_ground_mask (DESIGN f-13): struct sizes, the reference's error texts (checked before the
device is touched) and OB_NO_DEVICE without a GPU."""
import ctypes

import numpy as np

import __graft_entry__ as graft

ob = graft.load_package()
capi = ob._capi
lib = capi.lib


def test_structs_in_abi_sizeof_match_ctypes():
    for name, cls in {"ob_ground_model": capi.GroundModel, "ob_ground_item": capi.GroundItem}.items():
        assert lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name
    assert capi.OB_GROUND_FINAL == 7 and len(capi.GROUND_STAGES) == 8


def _item(h=2, w=3, n_returns=1, n_masks=1, mask_shape=None):
    """An item whose LUT handle is a placeholder: every check below fails before a handle is read."""
    rng = [np.zeros((h, w), np.uint32) for _ in range(n_returns)]
    masks = [np.full((h, w), 9, np.uint8) for _ in range(n_masks)]
    rp = (ctypes.c_void_p * max(n_returns, 1))(*[r.ctypes.data for r in rng])
    mp = (ctypes.c_void_p * max(n_masks, 1))(*[m.ctypes.data for m in masks])
    st, po = np.ones(w, np.uint32), np.zeros((w, 16))
    it = capi.GroundItem()
    it.lut, it.h, it.w, it.n_returns = 1, h, w, n_returns
    it.range = ctypes.cast(rp, ctypes.POINTER(ctypes.c_void_p)) if n_returns else None
    it.masks, it.n_masks = ctypes.cast(mp, ctypes.POINTER(ctypes.c_void_p)), n_masks
    it.mask_h, it.mask_w = mask_shape or (h, w)
    it.status, it.poses = st.ctypes.data, po.ctypes.data
    return it, (rng, masks, rp, mp, st, po)


def _call(it, grid_size=0.5):
    return lib.ob_ground_mask(ctypes.byref(it), 1, grid_size, capi.OB_GROUND_FINAL, None)


def test_error_texts_and_no_device():
    for grid in (0.0, -1.0, float("nan"), float("inf")):
        it, keep = _item()
        assert _call(it, grid) == capi.OB_INVALID_ARGUMENT
        assert lib.ob_last_error() == b"GroundSegConfig.grid_size must be > 0"
    it, keep = _item(n_returns=0)
    assert _call(it) == capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"frame must contain RANGE field for get_ground_mask"
    it, keep = _item(n_returns=2, n_masks=1)
    assert _call(it) == capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"not enough output masks provided for get_ground_mask_into"
    it, keep = _item(mask_shape=(2, 4))
    assert _call(it) == capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"output mask shape does not match frame shape"
    assert all((m == 9).all() for m in keep[1])
    if ob.core.device_count() == 0:
        it, keep = _item()
        assert _call(it) == capi.OB_NO_DEVICE
        assert all((m == 9).all() for m in keep[1])
