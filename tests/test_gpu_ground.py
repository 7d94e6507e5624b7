"""GPU checks of ground segmentation (DESIGN f-13): ob_ground_mask against the oracle (oracle/orc_ground.c) pass by
pass, bit for bit, given the same normals -- every grid after every pass, the model header and every mask pixel --
over the ray-cast scenes of tests/ground_scenes.py, the edge cases of the model, frame sets, host and device
buffers, refused calls and the launch count."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import ground as og
from oracle import oracle as orc
from tests import ground_scenes as gs

pytestmark = pytest.mark.gpu

ob = graft.load_package()
torch = pytest.importorskip("torch")
capi = ob._capi
GRIDS = ("valid", "obstacle", "floor_z", "height", "roughness")
HEADER = ("origin_x", "origin_y", "rows", "cols", "fallback_z", "footprint_bound", "valid", "has_columns")
c, s = np.cos(0.7), np.sin(0.7)
YAWED = np.array([[c, -s, 0, 3.0], [s, c, 0, -2.0], [0, 0, 1, 0.0], [0, 0, 0, 1]])  # as test_world_frame_pose

_cache = {}


def _frame(name, **kw):
    key = (name, tuple((k, str(v)) for k, v in sorted(kw.items())))
    if key not in _cache:
        f = gs.make_frame(name, **kw)
        f["lut"] = ob.core.XYZLutT.from_arrays(f["direction"], f["offset"], f["h"], f["w"])
        _cache[key] = f
    return _cache[key]


def _normals32(f, ranges=None):
    """The oracle's computed normals, rounded to float32 as a NORMALS field holds them."""
    ranges = f["ranges"] if ranges is None else ranges
    n = og.computed_normals(ranges[:2], f["direction"], f["offset"], f["poses"], f["sensor_to_body"])
    return [x.astype(np.float32) for x in n]


def _gpu_frame(f, ranges=None, normals=None, status=None, poses=None, lut=None):
    d = {"lut": lut or f["lut"], "ranges": f["ranges"] if ranges is None else ranges,
         "status": f["status"] if status is None else status, "poses": f["poses"] if poses is None else poses}
    if normals:
        d["normals"] = normals[0]
        d["normals2"] = normals[1] if len(normals) > 1 else None
    return d


def _oracle(f, d, stop=og.FINAL, grid_size=0.5):
    nrm = None
    if d.get("normals") is not None:
        nrm = [d["normals"].astype(np.float64)]
        if d.get("normals2") is not None:
            nrm.append(d["normals2"].astype(np.float64))
    return og.run(d["ranges"], d["status"], f["direction"], f["offset"], d["poses"], nrm, grid_size, stop)


def _host(x):
    return x.cpu().numpy() if torch.is_tensor(x) else x


def _assert_same(got, want_masks, want_model, want_grids, stop):
    for k in HEADER:
        a, b = got["model"][k], want_model[k]
        assert a == b or (np.isnan(a) and np.isnan(b)), (k, a, b)
        if isinstance(a, float):
            assert np.float64(a).tobytes() == np.float64(b).tobytes() or np.isnan(a), (k, a, b)
    if want_grids is None:
        assert got["grids"] is None
    else:
        for k in GRIDS:
            g = _host(got["grids"][k])
            w = want_grids[k]
            assert np.array_equal(g, w, equal_nan=True), (k, stop, int((g != w).sum()))
            if g.dtype == np.float64:  # the sign of zero too
                fin = np.isfinite(w)
                assert np.array_equal(np.signbit(g[fin]), np.signbit(w[fin])), (k, stop)
    masks = [_host(m) for m in got["masks"]]
    if stop == og.FINAL:
        for m, w in zip(masks, want_masks):
            assert np.array_equal(m, w), int((m != w).sum())
    else:
        assert all(not m.any() for m in masks)


def _compare_all_stops(f, d, grid_size=0.5, stops=range(og.FINAL + 1)):
    for stop in stops:
        got = ob.core.ground_mask([d], grid_size=grid_size, stop=stop, model=True)[0]
        masks, model, grids = _oracle(f, d, stop, grid_size)
        _assert_same(got, masks, model, grids, stop)
    return got


CASES = [(n, dual, pose) for n in gs.SCENES for dual in (False, True) for pose in ("identity", "yawed")]


@pytest.mark.parametrize("name,dual,pose", CASES)
def test_pass_by_pass(name, dual, pose):
    f = _frame(name, dual=dual, pose=None if pose == "identity" else YAWED)
    d = _gpu_frame(f, normals=_normals32(f))
    got = _compare_all_stops(f, d)
    assert got["model"]["valid"] == 1


@pytest.mark.parametrize("name", ["box_rooftop", "room"])
def test_pass_by_pass_128x2048(name):
    f = _frame(name, h=128, w=2048, dual=True)
    d = _gpu_frame(f, normals=_normals32(f))
    _compare_all_stops(f, d, stops=(og.STAGES.index("cells"), og.STAGES.index("prune"),
                                    og.STAGES.index("components"), og.FINAL))


def test_without_normals_and_normals_without_normals2():
    f = _frame("box_rooftop", dual=True)
    _compare_all_stops(f, _gpu_frame(f), stops=(og.FINAL,))
    n = _normals32(f)
    _compare_all_stops(f, _gpu_frame(f, normals=[n[0]]), stops=(og.FINAL,))


def test_third_return_is_classified_without_normals():
    f = _frame("wall", dual=True)
    ranges = f["ranges"] + [f["ranges"][0].copy()]
    d = _gpu_frame(f, ranges=ranges, normals=_normals32(f))
    got = _compare_all_stops(f, d, stops=(og.FINAL,))
    two = ob.core.ground_mask([_gpu_frame(f, normals=_normals32(f))], model=True)[0]
    for k in GRIDS:  # the third return leaves the model alone
        assert np.array_equal(_host(two["grids"][k]), _host(got["grids"][k]), equal_nan=True)
    assert len(got["masks"]) == 3


# ---- edges ----
def test_status_all_zero():
    f = _frame("flat")
    d = _gpu_frame(f, status=np.zeros(f["w"], np.uint32))
    got = _compare_all_stops(f, d, stops=(og.FINAL,))
    assert got["model"]["has_columns"] == 0 and got["grids"] is None


def test_one_column_without_returns():
    """The narrowest frame the LUT allows (a width-0 frame has no LUT): no point, masks written whole."""
    lut = ob.core.XYZLutT.from_arrays(np.ones((4, 3)), np.zeros((4, 3)), 4, 1)
    rng = np.zeros((4, 1), np.uint32)
    got = ob.core.ground_mask([{"lut": lut, "ranges": [rng], "status": np.ones(1, np.uint32),
                                "poses": np.eye(4).reshape(1, 16)}], model=True)[0]
    assert not got["masks"][0].any() and got["grids"] is None
    assert got["model"]["has_columns"] == 1 and got["model"]["rows"] == 0 and np.isnan(got["model"]["fallback_z"])


def test_all_points_closer_than_min_range():
    """Every point 0.1 m from a sensor at the world origin: no model point, the fallback classification."""
    f = _frame("flat")
    ranges = [np.where(f["ranges"][0] > 0, 100, 0).astype(np.uint32)]
    poses = np.repeat(np.eye(4).reshape(1, 16), f["w"], 0)
    got = _compare_all_stops(f, _gpu_frame(f, ranges=ranges, poses=poses), stops=(0, og.FINAL))
    assert got["model"]["rows"] == 0


def test_status_bit0_sets_the_span_and_nonzero_words_inside_count():
    f = _frame("ramp")
    st = np.zeros(f["w"], np.uint32)
    st[100] = 1
    st[900] = 1
    st[200:300] = 2  # inside the span: counted
    st[50:90] = 2    # outside the span: not counted
    _compare_all_stops(f, _gpu_frame(f, status=st), stops=(0, og.FINAL))


def test_non_finite_lut_entries():
    f = dict(_frame("tilted5"))
    d = f["direction"].copy()
    d[::7] = np.nan
    d[3::11, 2] = np.inf
    f["direction"] = d
    lut = ob.core.XYZLutT.from_arrays(d, f["offset"], f["h"], f["w"])
    _compare_all_stops(f, _gpu_frame(f, lut=lut), stops=(0, og.FINAL))


@pytest.mark.parametrize("grid_size", [0.05, 100.0])
def test_grid_sizes(grid_size):
    f = _frame("box_rooftop")
    _compare_all_stops(f, _gpu_frame(f, normals=_normals32(f)), grid_size=grid_size, stops=(0, 3, og.FINAL))


def test_one_far_point_makes_a_large_grid():
    f = dict(_frame("flat"))
    r = f["ranges"][0].copy()
    r[f["h"] // 2, 10] = 2_000_000  # 2 km away: a grid of millions of 0.5 m cells
    got = _compare_all_stops(f, _gpu_frame(f, ranges=[r]), stops=(0, og.FINAL))
    assert got["model"]["rows"] * got["model"]["cols"] > 1_000_000


def _synthetic(pts, h=4):
    """A frame whose points land exactly where chosen: one beam per column from the origin, range 1 m.  A point
    whose z is -0.0 gets it through negated zeros in its direction, offset and column pose."""
    w = len(pts)
    direction = np.zeros((h, w, 3))
    offset = np.zeros((h, w, 3))
    poses = np.repeat(np.eye(4).reshape(1, 16), w, 0)
    rng = np.zeros((h, w), np.uint32)
    rng[0] = 1000
    for k, (x, y, z) in enumerate(pts):
        direction[0, k] = (x * 0.001, y * 0.001, z * 0.001)
        if z == 0 and np.signbit(z):
            offset[0, k, 2] = -0.0
            poses[k].reshape(4, 4)[2] = (-0.0, -0.0, 1.0, -0.0)
    direction, offset = direction.reshape(-1, 3), offset.reshape(-1, 3)
    f = {"h": h, "w": w, "direction": direction, "offset": offset, "poses": poses,
         "status": np.ones(w, np.uint32), "ranges": [rng], "sensor_to_body": np.eye(4).reshape(16)}
    f["lut"] = ob.core.XYZLutT.from_arrays(direction, offset, h, w)
    return f


def test_two_components_of_equal_size():
    pts = []
    for x0 in (1.25, 6.25):  # two 3x3 patches far apart, same size; the second 0.8 m higher
        for i in range(3):
            for j in range(3):
                for _ in range(3):
                    pts.append((x0 + 0.5 * i, 1.25 + 0.5 * j, 0.0 if x0 < 5 else 0.8))
    f = _synthetic(pts)
    _compare_all_stops(f, _gpu_frame(f))


def test_signed_zero_heights_in_one_cell():
    pts = [(1.25, 1.25, z) for z in (0.0, -0.0, 0.0, -0.0, -0.0)] + [(1.75, 1.25, -0.0), (1.75, 1.25, 0.0)]
    f = _synthetic(pts)
    _, _, grids = og.run(f["ranges"], f["status"], f["direction"], f["offset"], f["poses"], stop=0)
    assert np.signbit(grids["height"][np.isfinite(grids["height"])]).any()  # the scene does hold a -0.0 height
    _compare_all_stops(f, _gpu_frame(f))


# ---- sets, memory kinds, refusals, launches ----
def test_set_of_two_sensors_with_empty_slots():
    a = _frame("box_rooftop", dual=True)
    b = _frame("room", h=32, w=512, seed=5)
    da, db = _gpu_frame(a, normals=_normals32(a)), _gpu_frame(b)
    got = ob.core.ground_mask([None, da, None, db, None], model=True)
    assert got[0] is None and got[2] is None and got[4] is None
    for f, d, g in ((a, da, got[1]), (b, db, got[3])):
        masks, model, grids = _oracle(f, d)
        _assert_same(g, masks, model, grids, og.FINAL)
        one = ob.core.ground_mask([d])[0]
        for m1, m2 in zip(one["masks"], g["masks"]):
            assert np.array_equal(m1, m2)


def test_device_buffers():
    f = _frame("wall", dual=True)
    n = _normals32(f)
    dd = {"lut": f["lut"], "ranges": [torch.from_numpy(r.astype(np.int64)).to(torch.int32).cuda() for r in f["ranges"]],
          "status": torch.from_numpy(f["status"].astype(np.int32)).cuda(),
          "poses": torch.from_numpy(f["poses"]).cuda(), "normals": torch.from_numpy(n[0]).cuda(),
          "normals2": torch.from_numpy(n[1]).cuda()}
    got = ob.core.ground_mask([dd], stop=og.FINAL, model=True)[0]
    assert got["masks"][0].is_cuda and got["grids"]["height"].is_cuda
    masks, model, grids = _oracle(f, _gpu_frame(f, normals=n))
    _assert_same(got, masks, model, grids, og.FINAL)


def _raw_item(f, masks, n_masks=None, mask_shape=None):
    item = capi.GroundItem()
    rp = (C.c_void_p * len(f["ranges"]))(*[r.ctypes.data for r in f["ranges"]])
    mp = (C.c_void_p * len(masks))(*[m.ctypes.data for m in masks])
    item.lut, item.h, item.w, item.n_returns = f["lut"]._h, f["h"], f["w"], len(f["ranges"])
    item.range = C.cast(rp, C.POINTER(C.c_void_p))
    item.masks = C.cast(mp, C.POINTER(C.c_void_p))
    item.n_masks = len(masks) if n_masks is None else n_masks
    item.mask_h, item.mask_w = mask_shape or (f["h"], f["w"])
    item.status, item.poses = f["status"].ctypes.data, f["poses"].ctypes.data
    return item, (rp, mp)


def test_refused_calls_write_nothing():
    f = _frame("flat", dual=True)
    st = ob.core._stream(None)
    masks = [np.full((f["h"], f["w"]), 9, np.uint8) for _ in range(2)]
    cases = [
        (dict(), 0.0, "GroundSegConfig.grid_size must be > 0"),
        (dict(), float("nan"), "GroundSegConfig.grid_size must be > 0"),
        (dict(n_masks=1), 0.5, "not enough output masks provided for get_ground_mask_into"),
        (dict(mask_shape=(f["h"], f["w"] + 1)), 0.5, "output mask shape does not match frame shape"),
    ]
    for kw, grid, text in cases:
        item, keep = _raw_item(f, masks, **kw)
        assert capi.lib.ob_ground_mask(C.byref(item), 1, grid, capi.OB_GROUND_FINAL, st.h) == capi.OB_INVALID_ARGUMENT
        assert capi.lib.ob_last_error().decode() == text
    item, keep = _raw_item(f, masks)
    item.n_returns = 0
    assert capi.lib.ob_ground_mask(C.byref(item), 1, 0.5, capi.OB_GROUND_FINAL, st.h) == capi.OB_INVALID_ARGUMENT
    assert capi.lib.ob_last_error().decode() == "frame must contain RANGE field for get_ground_mask"
    # a grid output shorter than the grid: refused after the shape wait, nothing written
    item, keep = _raw_item(f, masks)
    hv = np.full(4, 5.0)
    item.height, item.grid_capacity = hv.ctypes.data, 4
    assert capi.lib.ob_ground_mask(C.byref(item), 1, 0.5, capi.OB_GROUND_FINAL, st.h) == capi.OB_INVALID_ARGUMENT
    assert capi.lib.ob_last_error().decode() == "output capacity too small"
    st.sync()
    assert all((m == 9).all() for m in masks) and (hv == 5.0).all()
    # an f32 lut is refused
    lut32 = ob.core.XYZLutT.from_arrays(f["direction"].astype(np.float32), f["offset"].astype(np.float32), f["h"],
                                        f["w"])
    item, keep = _raw_item(f, masks)
    item.lut = lut32._h
    assert capi.lib.ob_ground_mask(C.byref(item), 1, 0.5, capi.OB_GROUND_FINAL, st.h) == capi.OB_INVALID_ARGUMENT
    assert capi.lib.ob_last_error().decode() == "ground segmentation needs a float64 lut"
    st.sync()
    assert all((m == 9).all() for m in masks)


def test_launches_do_not_depend_on_the_number_of_frames():
    f = _frame("flat", h=16, w=256)
    d = _gpu_frame(f)
    counts = {}
    for n in (1, 16):
        ob.core.ground_mask([d] * n)
        before = {k: ob.core.kernel_launch_count(k) for k in ("ground", "normals")}
        total = ob.core.kernel_launch_count()
        ob.core.ground_mask([d] * n)
        counts[n] = ({k: ob.core.kernel_launch_count(k) - v for k, v in before.items()},
                     ob.core.kernel_launch_count() - total)
    assert counts[1] == counts[16]
    assert counts[1][0]["ground"] == 22 and counts[1][0]["normals"] == 0 and counts[1][1] == 22


@pytest.mark.parametrize("name", ["flat", "box_rooftop", "room"])
def test_truth_thresholds(name):
    """The thresholds of test_oracle_ground.py hold for the GPU masks."""
    f = _frame(name)
    m = ob.core.ground_mask([_gpu_frame(f, normals=_normals32(f))])[0]["masks"][0].astype(bool)
    ground, obj = gs.truth_sets(f)
    assert m[ground].mean() >= 0.99
    if obj.any():
        assert (~m[obj]).mean() >= 0.99


# ---- computed normals ----
def _oracle_normals(f, subtent):
    """get_ground_mask's normals, from the normals oracle given the vertical subtent the GPU used."""
    origins = og.sensor_origins(f["poses"], f["sensor_to_body"])
    p = [og.dewarped_points(r, f["direction"], f["offset"], f["poses"]) for r in f["ranges"][:2]]
    if len(p) == 2:
        return list(orc.normals(p[0], f["ranges"][0], p[1], f["ranges"][1], sensor_origins_xyz=origins,
                                vertical_subtent=subtent))
    return [orc.normals(p[0], f["ranges"][0], sensor_origins_xyz=origins, vertical_subtent=subtent)]


@pytest.mark.parametrize("name,dual,pose", [("box_rooftop", True, "yawed"), ("room", False, "identity"),
                                            ("wall", True, "identity")])
def test_computed_normals(name, dual, pose):
    f = _frame(name, dual=dual, pose=None if pose == "identity" else YAWED)
    d = _gpu_frame(f)
    d["sensor_to_body"] = f["sensor_to_body"]
    got = ob.core.ground_mask([d], model=True)[0]
    s = got["vertical_subtent"]
    assert s > 0
    nrm = _oracle_normals(f, s)
    masks, model, grids = og.run(f["ranges"], f["status"], f["direction"], f["offset"], f["poses"], nrm)
    _assert_same(got, masks, model, grids, og.FINAL)
    # the oracle's own subtent (host acos) may differ in the last bits: count the pixels that then differ
    own, _, _ = og.run(f["ranges"], f["status"], f["direction"], f["offset"], f["poses"],
                       og.computed_normals(f["ranges"][:2], f["direction"], f["offset"], f["poses"],
                                           f["sensor_to_body"]))
    diff = sum(int((_host(m) != w).sum()) for m, w in zip(got["masks"], own))
    print(f"computed normals, {name}: {diff} mask pixels differ from the oracle deriving its own subtent")
    assert diff <= 0.001 * f["h"] * f["w"]


def test_computed_normals_launches_do_not_depend_on_the_number_of_frames():
    f = _frame("flat", h=16, w=256, dual=True)
    d = dict(_gpu_frame(f), sensor_to_body=f["sensor_to_body"])
    counts = {}
    for n in (1, 16):
        ob.core.ground_mask([d] * n)
        before = {k: ob.core.kernel_launch_count(k) for k in ("ground", "normals")}
        ob.core.ground_mask([d] * n)
        counts[n] = {k: ob.core.kernel_launch_count(k) - v for k, v in before.items()}
    assert counts[1] == counts[16] == {"ground": 23, "normals": 3}


def test_width_zero_through_the_c_abi():
    """An item of width 0 has no pixel: the call succeeds and neither reads its LUT (a LUT cannot be 0 wide; a 1 x 1
    handle stands in) nor writes anything."""
    lut = ob.core.XYZLutT.from_arrays(np.ones((1, 3)), np.zeros((1, 3)), 1, 1)
    item = capi.GroundItem()
    rng = np.zeros(1, np.uint32)
    rp = (C.c_void_p * 1)(rng.ctypes.data)
    mp = (C.c_void_p * 1)(None)
    item.lut, item.h, item.w, item.n_returns = lut._h, 1, 0, 1
    item.range, item.masks, item.n_masks = C.cast(rp, C.POINTER(C.c_void_p)), C.cast(mp, C.POINTER(C.c_void_p)), 1
    item.mask_h, item.mask_w = 1, 0
    st = ob.core._stream(None)
    model = capi.GroundModel()
    model.rows = 99
    item.model = C.addressof(model)
    assert capi.lib.ob_ground_mask(C.byref(item), 1, 0.5, capi.OB_GROUND_FINAL, st.h) == capi.OB_OK
    st.sync()
    assert model.rows == 99
    # a LUT of another shape is refused
    stt, poses = np.ones(2, np.uint32), np.zeros((2, 16))
    item.w, item.mask_w, item.status, item.poses = 2, 2, stt.ctypes.data, poses.ctypes.data
    assert capi.lib.ob_ground_mask(C.byref(item), 1, 0.5, capi.OB_GROUND_FINAL, st.h) == capi.OB_INVALID_ARGUMENT
    assert capi.lib.ob_last_error() == b"lut shape does not match frame shape"


# ---- GroundSegEngine ----
def _engine_scans(device):
    """Two dual-return scans and an empty slot of a sensor 1.8 m above the `box_rooftop` scene's ground plane,
    ray-cast along the sensor's own LUT; the second scan has no RANGE2 but a stale GROUND2."""
    pyapi = ob.pyapi
    h, w = 32, 512
    info = ob.SensorInfo("RNG19_RFL8_SIG16_NIR16_DUAL", h, w, fw_rev="v3.2.1", sn=7)
    alt = np.linspace(11.0, -11.0, h)
    info.set_intrinsics(np.zeros(h), alt, np.eye(4), np.eye(4))
    lut = pyapi.XYZLut(info)._lut
    dvec = np.asarray(lut.direction).reshape(h, w, 3)
    unit = dvec / np.linalg.norm(dvec, axis=-1, keepdims=True)
    scene = gs.Scene(gs.flat, boxes=[(10.0, 12.0, 2.0, 4.0, 0.0, 1.0)])
    t, label = scene.cast(unit, np.array([0.0, 0.0, 0.0]) + np.array([0.0, 0.0, 1.8]))
    rng = np.where(np.isfinite(t), np.round(t * 1000.0), 0).astype(np.uint32)
    scans = []
    for k in range(2):
        sc = pyapi.LidarScan(info)
        sc.field("RANGE")[:] = rng
        sc.status[:] = 1
        sc.body_to_world[:] = np.eye(4)
        sc.body_to_world[:, 2, 3] = 1.8
        if k == 0:
            sc.field("RANGE2")[:] = np.where(np.arange(w)[None, :] % 9 == 0, rng, 0)
            sc.add_field("GROUND", np.uint8)
            sc.field("GROUND")[:] = 5
        else:
            sc.del_field("RANGE2")
            sc.add_field("GROUND2", np.uint8)
        scans.append(sc)
    ds = None
    if device:
        ds = []
        for sc in scans:
            d = pyapi.DeviceLidarScan(info)
            d.host.status[:] = sc.status
            d.host.body_to_world[:] = sc.body_to_world
            for name in list(d._fields):
                if name not in sc.fields:
                    del d._fields[name]
            for name in sc.fields:
                a = sc.field(name)
                d._fields[name] = torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a.copy()).cuda()
            ds.append(d)
    z = 1.8 + np.where(np.isfinite(t), t, 0.0) * unit[..., 2]
    return info, lut, scans, ds, label, z


@pytest.mark.parametrize("device", [False, True])
def test_engine_update(device):
    pyapi = ob.pyapi
    with pytest.raises(ValueError, match="GroundSegConfig.grid_size must be > 0"):
        pyapi.GroundSegEngine.create(pyapi.GroundSegConfig(0.0))
    info, lut, scans, ds, label, z = _engine_scans(device)
    frames = [ds[0], None, ds[1]] if device else [scans[0], None, scans[1]]
    eng = pyapi.GroundSegEngine.create(pyapi.GroundSegConfig())
    assert eng.update(frames) is frames
    f0, f2 = frames[0], frames[2]
    assert "GROUND" in f0.fields and "GROUND2" in f0.fields
    assert "GROUND" in f2.fields and "GROUND2" not in f2.fields
    # the same call through core.ground_mask with the engine's LUT and computed normals
    for sc, fr in ((scans[0], f0), (scans[1], f2)):
        ranges = [sc.field("RANGE")] + ([sc.field("RANGE2")] if "RANGE2" in sc.fields else [])
        want = ob.core.ground_mask([{"lut": lut, "ranges": ranges, "status": sc.status, "poses": sc.body_to_world,
                                     "sensor_to_body": np.eye(4)}])[0]["masks"]
        for ret, m in enumerate(want):
            g = fr.field(pyapi._return_field_name("GROUND", ret))
            assert (g.is_cuda if device else True)
            assert np.array_equal(_host(g), m)
    g = _host(f0.field("GROUND")).astype(bool)
    rng = scans[0].field("RANGE")
    ground = (label == 1) & (rng > 0)
    obj = (label == 2) & (rng > 0) & (z > 0.5)  # object pixels more than 0.5 m above the ground
    assert ground.sum() > 1000 and g[ground].mean() >= 0.99
    assert obj.any() and (~g[obj]).mean() >= 0.99


def test_cpp_dropin_example(tmp_path):
    import os
    import subprocess
    graft.build()
    root = graft.ROOT
    lib_dir = os.path.join(root, "ouster-sdk_b200", "lib")
    exe = str(tmp_path / "ground_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "ground_dropin_example.cpp"), "-L", lib_dir,
                           "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    out = subprocess.run([exe, "gpu"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "GROUND DROPIN GPU OK" in out.stdout, (out.stdout, out.stderr)
