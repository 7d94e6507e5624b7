"""CPU tests of the frame operations oracle (oracle/orc_frame_ops.c, oracle/frame_ops.py) and of the host-side
parts of ouster_sdk_b200.frame_ops that need no GPU (product-line rewriting, index rules, error texts)."""
import ctypes
import glob
import json
import os

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import frame_ops as ofo
from oracle import oracle as orc

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _frame(h=16, w=64, seed=0, dual=True):
    rs = np.random.default_rng(seed)
    f = ofo.Frame(h, w, rs.integers(-30, 31, h))
    f.add("RANGE", rs.integers(0, 20000, (h, w), dtype=np.uint32))
    f.add("SIGNAL", rs.integers(0, 1 << 16, (h, w), dtype=np.uint16))
    f.add("REFLECTIVITY", rs.integers(0, 256, (h, w), dtype=np.uint8))
    if dual:
        f.add("RANGE2", rs.integers(0, 20000, (h, w), dtype=np.uint32))
        f.add("SIGNAL2", rs.integers(0, 1 << 16, (h, w), dtype=np.uint16))
    return f


@pytest.mark.parametrize("w", [8, 64, 512, 1024, 2048])
def test_direct_filter_uv_v_equals_destagger_mask_stagger(w):
    rs = np.random.default_rng(w)
    h = 12
    for trial in range(4):
        shifts = rs.integers(-30, 31, h).astype(np.int32)
        lo = int(rs.integers(0, w))
        hi = int(rs.integers(lo, w + 1))
        a = rs.integers(1, 1000, (h, w)).astype(np.uint32)
        lit = a.copy()
        assert ofo.lib().orc_fo_uv_v_literal(lit.ctypes.data, 3, 4, shifts.ctypes.data, h, w, lo, hi, 0.0) == 0
        direct = np.where(ofo.uv_v_mask(shifts, h, w, lo, hi) == 0, 0, a).astype(np.uint32)
        assert np.array_equal(lit, direct), (trial, lo, hi)
        # the literal form is what destagger -> mask -> stagger gives through the project oracle's destagger
        d = orc.destagger(a, shifts)
        d[:, lo:hi] = 0
        assert np.array_equal(orc.destagger(d, shifts, inverse=True), lit)


def test_reference_python_assertions_on_synthetic_frames():
    f = _frame()
    # test_select: selected rows equal the source rows
    s = ofo.select_rows(f, [1, 5, 7])
    assert np.array_equal(s.field("RANGE"), f.field("RANGE")[[1, 5, 7]])
    # test_mask: half masked
    g = f.copy()
    m = np.ones((f.h, f.w), np.uint8)
    m[:, : f.w // 2] = 0
    ofo.mask(g, ["RANGE"], m)
    assert np.count_nonzero(g.field("RANGE")[:, : f.w // 2]) == 0
    assert np.array_equal(g.field("RANGE")[:, f.w // 2:], f.field("RANGE")[:, f.w // 2:])
    # test_clip: max == upper, non-zero min == lower
    g = f.copy()
    ofo.clip(g, ["RANGE"], 1000, 5000)
    r = g.field("RANGE")
    assert r.max() <= 5000 and r[r > 0].min() >= 1000
    g.field("RANGE")[0, :2] = [1000, 5000]
    ofo.clip(g, ["RANGE"], 1000, 5000)
    assert r.max() == 5000 and r[r > 0].min() == 1000
    # test_reduce: h == beams
    s = ofo.select_rows(f, list(range(0, f.h, 4)))
    assert s.field("RANGE").shape[0] == f.h // 4


def test_filter_xyz_dewarp_points_changes_spatial_mask():
    """test_filter_xyz_dewarp_points_changes_spatial_mask: no pixel lies in the body-frame band, half the pixels
    (the columns posed into it) lie in the world-frame band."""
    h, w = 8, 32
    f = ofo.Frame(h, w)
    f.add("RANGE", np.full((h, w), 1000, np.uint32))
    d = np.zeros((h * w, 3))
    d[:, 0] = 0.001
    o = np.zeros((h * w, 3))
    poses = np.tile(np.eye(4), (w, 1, 1))
    poses[w // 2:, 2, 3] = 10.0
    body = orc.cartesian(f.field("RANGE"), d, o).reshape(h, w, 3)
    world = orc.dewarp(body, poses)
    g = f.copy()
    ofo.filter_xyz(g, lambda n: body, 2, 5.0, 15.0)
    assert np.count_nonzero(g.field("RANGE") == 0) == 0
    ofo.filter_xyz(g, lambda n: world, 2, 5.0, 15.0)
    assert np.count_nonzero(g.field("RANGE") == 0) == h * w // 2


def test_filter_field_is_inside_and_reads_source_before_writing():
    f = _frame(seed=3)
    g = f.copy()
    ofo.filter_field(g, "RANGE", 5000, 10000, 0, ["RANGE", "SIGNAL"])
    inside = (f.field("RANGE") >= 5000) & (f.field("RANGE") <= 10000)
    assert np.all(g.field("RANGE")[inside] == 0) and np.array_equal(g.field("RANGE")[~inside], f.field("RANGE")[~inside])
    assert np.all(g.field("SIGNAL")[inside] == 0)
    assert np.array_equal(g.field("REFLECTIVITY"), f.field("REFLECTIVITY"))


def test_clip_nan_and_u64_rounding():
    f = ofo.Frame(1, 4)
    a = f.add("F", np.array([[np.nan, 1.0, -np.inf, 3.0]], np.float32))
    ofo.clip(f, [], 0.0, 2.0, 7.0)
    assert np.array_equal(a, np.array([[7, 1, 7, 7]], np.float32))
    f = ofo.Frame(1, 2)
    # 2**53 + 1 rounds to 2**53 in double, so it is inside [0, 2**53]
    u = f.add("U", np.array([[2 ** 53 + 1, 2 ** 53 + 3]], np.uint64))
    ofo.clip(f, [], 0.0, float(2 ** 53), 0)
    assert u[0, 0] == 2 ** 53 + 1 and u[0, 1] == 0


def test_error_texts():
    f = _frame(dual=False)
    f.add("IMU", np.zeros(f.w, np.float64), field_class=ofo.COLUMN_FIELD)
    f.add("EXTRA", np.zeros((f.h, f.w, 3), np.uint16))
    with pytest.raises(ValueError, match=r"^Only PIXEL_FIELD frame fields are supported here; requested non-pixel "
                                         r"fields: \[IMU\]$"):
        ofo.clip(f, ["RANGE", "IMU"], 0, 1)
    with pytest.raises(ValueError, match=r"fields: \['IMU'\]$"):
        ofo.filter_xyz(f, lambda n: np.zeros((f.h, f.w, 3)), 0, filtered_fields=["IMU"])
    with pytest.raises(ValueError, match=r"^Field: Eigen array conversion failed due to dimension mismatch\. "
                                         r"Underlying data has 3 dimensions but must have 2 dimensions\.$"):
        ofo.clip(f, ["EXTRA"], 0, 1)
    with pytest.raises(ValueError, match=r"^filter_field requires a pixel field with shape \(h, w\) to build a mask$"):
        ofo.filter_field(f, "EXTRA", 0, 1)
    with pytest.raises(ValueError, match=r"^coord_2d == x must be either 'u' or 'v'$"):
        ofo.filter_uv(f, "x", 0, 1)
    with pytest.raises(ValueError, match=r"^lower == 0 and upper == 17 must be in the range \[0, 16\]$"):
        ofo.filter_uv(f, "u", 0, 17)
    with pytest.raises(ValueError, match=r"^lower == 3 must be less than upper == 2$"):
        ofo.filter_uv(f, "u", 3, 2)
    with pytest.raises(ValueError, match=r"^Used mask size doesn't match frame size$"):
        ofo.mask(f, [], np.ones((2, 2), np.uint8))
    with pytest.raises(ValueError, match="invalid value cannot be represented"):
        ofo.clip(f, ["RANGE"], 0, 1, -1)


def test_python_layer_texts_and_index_rules():
    ob = graft.load_package()
    fo = ob.frame_ops
    with pytest.raises(ValueError, match=r"^beam indices can't be empty$"):
        fo._validate_beam_indices([], 4)
    with pytest.raises(ValueError, match=r"^beam indices can't contain duplicates$"):
        fo._validate_beam_indices([1, 1], 4)
    with pytest.raises(ValueError, match=r"^beam indices \[4, 9\] must be in the range \[0, 4\)$"):
        fo._validate_beam_indices([0, 4, 9], 4)
    with pytest.raises(ValueError, match=r"^factor == 0 can't be negative$"):
        fo.reduce_factor_to_indices(0, 8)
    with pytest.raises(ValueError, match=r"^factor == 3 must be a divisor of 8$"):
        fo.reduce_factor_to_indices(3, 8)
    assert fo.reduce_factor_to_indices(8, 8) == [4]
    assert fo.reduce_factor_to_indices(2, 8) == [0, 2, 4, 6]
    with pytest.raises(ValueError, match=r"^axis_idx == 3 must be in the range \[0, 2\]$"):
        fo.filter_xyz(None, None, 3)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "*.json"))))
def test_prod_line_rewriting(path):
    ob = graft.load_package()
    meta = json.load(open(path))
    if "prod_line" not in meta:
        pytest.skip("fixture without a product line")
    pl = meta["prod_line"]
    pi = ob.frame_ops.product_info(pl)
    ff = pi["form_factor"]
    assert ff.startswith("OS") and pi["beam_count"] in (32, 128)
    out = ob.frame_ops.form_factor_prod_line(pl, 64)
    assert out == "OS-" + ff[2] + "-64", (pl, out)
    assert ob.frame_ops.form_factor_prod_line("OS-0-128-U1", 8) == "OS-0-8"
    assert ob.frame_ops.form_factor_prod_line("OS-DOME-128", 32) == "OSDOME-32"
    assert ob.frame_ops.form_factor_prod_line("OS-1-MAX-128", 64) == "OS1MAX-64"
    assert ob.frame_ops.form_factor_prod_line("OS-1-64-RGB", 16) == "OS-1-16-RGB"
    assert ob.frame_ops.form_factor_prod_line("", 16) == "-16"
    with pytest.raises(RuntimeError, match=r'^Product Info "\?\?" is not a recognized product info$'):
        ob.frame_ops.product_info("??")


def test_abi_struct_layouts():
    ob = graft.load_package()
    capi = ob._capi
    for name, cls in {"ob_frame_field": capi.FrameField, "ob_frame_ops_io": capi.FrameOpsIO,
                      "ob_frame_rows_entry": capi.FrameRowsEntry, "ob_frame_rows_io": capi.FrameRowsIO}.items():
        assert capi.lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name
