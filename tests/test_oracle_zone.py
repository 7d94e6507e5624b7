"""CPU tests of the zone-monitoring oracle (oracle/orc_zone.c) and the host side of the zone API: the reference's
known answers, the golden rendered ZRB, Mesh's STL parser on every fixture, and the error texts."""
import ctypes
import json
import os
import re
import struct

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import zone as oz

ZDIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zone")


def sensor_meta(name):
    """the fields BeamConfig reads from a sensor metadata JSON"""
    m = json.load(open(os.path.join(ZDIR, name)))
    fmt, bi = m["lidar_data_format"], m["beam_intrinsics"]
    return {"w": fmt["columns_per_frame"], "h": fmt["pixels_per_column"],
            "beam_to_lidar_transform": np.array(bi["beam_to_lidar_transform"], np.float64).reshape(4, 4),
            "lidar_to_sensor_transform": np.array(m["lidar_intrinsics"]["lidar_to_sensor_transform"],
                                                  np.float64).reshape(4, 4),
            "beam_azimuth_angles": bi["beam_azimuth_angles"], "beam_altitude_angles": bi["beam_altitude_angles"],
            "sn": int(m["sensor_info"]["prod_sn"])}


def stl_tris(name):
    b = open(os.path.join(ZDIR, name), "rb").read()
    n = struct.unpack_from("<I", b, 80)[0]
    return np.array([np.frombuffer(b, "<f4", 12, 84 + 50 * i)[3:] for i in range(n)], np.float32)


def read_zrb(path):
    """(m_per_zmbin, [beam_to_lidar, lidar_to_sensor, sensor_to_body], payload (h, w) uint32): the header's
    transforms are stored column-major, the payload column by column, far bins in the high 16 bits"""
    b = open(path, "rb").read()
    ncols, nrows = struct.unpack_from("<II", b, 55)
    mpb = struct.unpack_from("<f", b, 63)[0]
    mats = [np.frombuffer(b, "<f4", 16, 131 + 64 * k).reshape(4, 4).T.astype(np.float64) for k in range(3)]
    pay = np.frombuffer(b, "<u4", nrows * ncols, 579).reshape(ncols, nrows).T
    return mpb, mats, pay


def s2b_z1():
    m = np.eye(4)
    m[2, 3] = 1.0
    return m


def test_known_answer_max_counts():
    """test_emulated_zone_mon_init: max_counts == {0: 12096, 1: 3098} (785.json, BODY, sensor_to_body z = 1 m)"""
    meta = sensor_meta("785.json")
    (bd, bo), _ = oz.beam_luts(meta, s2b_z1())
    got = {}
    for i in (0, 1):
        near, far, _ = oz.render(stl_tris(f"{i}.stl"), bd, bo, meta["h"], meta["w"])
        got[i] = int(np.count_nonzero(near < far))
    assert got == {0: 12096, 1: 3098}


def test_known_answer_get_packet():
    """test_emulated_zone_mon_get_packet: count 1218 at a constant 1000 mm, min = max = mean = 1000, triggered"""
    meta = sensor_meta("OS-0-128_v3.0.1_1024x10.2.json")
    (bd, bo), _ = oz.beam_luts(meta, np.eye(4))
    near, far, _ = oz.render(stl_tris("0.stl"), bd, bo, meta["h"], meta["w"])
    rng = np.full((meta["h"], meta["w"]), 1000, np.uint32)
    bm = np.zeros_like(rng)
    c = oz.counts(rng, near, far, 0, bm)
    assert c["count"] == 1218
    assert c["min_range"] == c["max_range"] == c["mean_range"] == 1000
    assert np.count_nonzero(bm) == 1218 and set(np.unique(bm)) == {0, 1}
    triggers, alerts = oz.trigger(1, 1, 1, c["count"], 0, 0)
    assert (triggers, alerts) == (1, 1)  # trigger_status 1, triggered_frames 1


def test_golden_zrb():
    """0.zrb, quantised as Zrb::save does (float(mm) / float(mm_per_bin), std::round): every near bin equal, every far
    bin equal except one ray, (75, 211), which the file's producer rounded from slightly different arithmetic"""
    mpb, (b2l, l2s, s2b), pay = read_zrb(os.path.join(ZDIR, "0.zrb"))
    meta = sensor_meta("785.json")
    assert np.allclose(b2l, meta["beam_to_lidar_transform"], atol=1e-4)
    assert np.array_equal(s2b, s2b_z1())
    (bd, bo), _ = oz.beam_luts(meta, s2b)
    near, far, hits = oz.render(stl_tris("0.stl"), bd, bo, meta["h"], meta["w"])
    mm_per_bin = np.float32(mpb) * np.float32(1000)
    q = lambda a: np.round(a.astype(np.float32) / mm_per_bin).astype(np.uint32)
    assert np.array_equal(q(near), pay & 0xFFFF)
    bad = np.argwhere(q(far) != pay >> 16).tolist()
    assert bad == [[75, 211]]
    assert q(far)[75, 211] == 412 and (pay >> 16)[75, 211] == 413
    # one hit ray has near == far: two triangles hit at the same t (a shared edge)
    assert hits == 12097 and np.count_nonzero(near < far) == 12096
    assert np.count_nonzero((near == far) & (far > 0)) == 1


def test_mesh_regressions():
    """mesh_test.cpp: closest_and_farthest_intersections and bounding_sphere known values"""
    ok, (n, f) = oz.closest_and_farthest(stl_tris("0.stl"), [0.00397694, 0.000619036, 1.0436],
                                         [-0.0914688, 0.975646, -0.199368])
    assert ok
    assert abs(n - 2.02771592) <= 4 * np.spacing(np.float32(2.0277)) and abs(f - 2.65380812) <= 4 * np.spacing(
        np.float32(2.65))
    tris = np.array([[1] * 9, [2] * 9, [2] * 9], np.float32)
    c, r = oz.bounding_sphere(tris)
    assert np.allclose(c, 1.666667) and np.isclose(r, 1.1547004)


def test_intersect_rules():
    tri = np.array([0, 0, 5, 1, 0, 5, 0, 1, 5], np.float32)
    assert oz.tri_intersect(tri, [0.1, 0.1, 0], [0, 0, 1]) == pytest.approx(5.0)
    assert oz.tri_intersect(tri, [0.1, 0.1, 10], [0, 0, 1]) == pytest.approx(-5.0)  # behind: never counted
    assert oz.tri_intersect(tri, [0.1, 0.1, 0], [1, 0, 0]) == -np.finfo(np.float32).max  # parallel
    nan_tri = tri.copy()
    nan_tri[0] = np.nan
    assert np.isnan(oz.tri_intersect(nan_tri, [0.1, 0.1, 0], [0, 0, 1]))  # NaN passes every rejection
    ok, _ = oz.closest_and_farthest(nan_tri, [0.1, 0.1, 0], [0, 0, 1])
    assert not ok


def test_render_errors():
    d = np.tile([0.0, 0.0, 0.001], (4, 1))
    o = np.zeros((4, 3))
    far_tri = np.array([-1e7, -1e7, 5e6, 1e7, -1e7, 5e6, 0, 1e7, 5e6], np.float32)
    with pytest.raises(RuntimeError, match=r"^Zone::render: range overflow$"):
        oz.render(far_tri, d, o, 2, 2)
    tri = np.array([-1, -1, 5, 1, -1, 5, 0, 1, 5], np.float32)
    with pytest.raises(RuntimeError, match=r"^Zone: area of rendered zone \(4\) is smaller than point_count \(5\) "
                                           r"specified in zone\.$"):
        oz.render(tri, d, o, 2, 2, point_count=5)
    near, far, px = oz.render(tri, d, o, 2, 2, point_count=4)
    assert px == 4 and np.all(near == 0) and np.all(far == 5000)


def test_trigger_state_machine():
    seq = [5, 5, 0, 5, 5, 5]
    t = a = 0
    got = []
    for c in seq:
        t, a = oz.trigger(1, 3, 2, c, t, a)
        got.append((t, a))
    assert got == [(1, 0), (2, 1), (0, 0), (1, 0), (2, 1), (3, 2)]
    assert oz.trigger(2, 3, 1, 2, 0, 0) == (1, 1)   # VACANCY: count < point_count
    assert oz.trigger(2, 3, 1, 3, 4, 4) == (0, 0)


@pytest.fixture(scope="module")
def ob():
    graft.build()
    return graft.load_package()


def test_abi_zone_structs(ob):
    capi = ob._capi
    for name, cls in (("ob_zone_desc", capi.ZoneDesc), ("ob_zone_render_io", capi.ZoneRenderIO),
                      ("ob_zone_live", capi.ZoneLive), ("ob_zone_state", capi.ZoneState)):
        assert capi.lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name
    assert ctypes.sizeof(capi.ZoneState) == 37 == ob.core.ZONE_STATE_DTYPE.itemsize


@pytest.mark.parametrize("name,n", [("0.stl", 12), ("1.stl", 12), ("ascii.stl", 12), ("solidworks_binary.stl", 12),
                                    ("empty.stl", 0), ("plane.stl", 2), ("tiny.stl", None)])
def test_stl_parser_accepts(ob, name, n):
    m = ob.pyapi.Mesh()
    assert m.load_from_stl(os.path.join(ZDIR, name))
    if n is not None:
        assert len(m.triangles) == n
    if name.endswith("0.stl") or name == "solidworks_binary.stl":
        assert np.array_equal(m.triangles.reshape(-1, 9), stl_tris(name))


def test_stl_ascii_values(ob):
    m = ob.pyapi.Mesh()
    assert m.load_from_stl(os.path.join(ZDIR, "ascii.stl"))
    assert np.array_equal(m.triangles[0], [[-20, -20, 40], [20, -20, 40], [-20, 20, 40]])


@pytest.mark.parametrize("name", ["ascii_invalid_expected_vertex.stl", "ascii_invalid_expected_endloop.stl",
                                  "ascii_invalid_expected_outer_loop.stl", "ascii_invalid_expected_endfacet.stl",
                                  "ascii_empty.stl", "ascii_invalid_expected_solid.stl",
                                  "ascii_invalid_expected_endsolid.stl", "ascii_invalid_unexpected_line.stl"])
def test_stl_parser_rejects(ob, name):
    assert not ob.pyapi.Mesh().load_from_stl(os.path.join(ZDIR, name))


def test_stl_binary_edges(ob):
    load = ob.pyapi.load_stl_triangles
    rec = struct.pack("<12fH", 0, 0, 1, *range(9), 0)
    assert load(b"\0" * 80 + struct.pack("<I", 1) + rec).shape == (1, 3, 3)
    assert load(b"\0" * 80 + struct.pack("<I", 1) + rec[:48]).shape == (1, 3, 3)  # attribute bytes may be cut
    assert load(b"\0" * 80 + struct.pack("<I", 2) + rec + rec[:47]) is None
    assert load(b"\0" * 79) is None
    assert load(b"\0" * 80) is None
    # "endsolid" inside the header does not make a file ASCII
    assert load(b"solid x endsolid".ljust(80, b" ") + struct.pack("<I", 0)).shape == (0, 3, 3)


def test_zone_invariant_texts(ob):
    api = ob.pyapi
    z = api.Zone()
    for setup, text in ((lambda: None, "Zone: point_count must be in [1, 262143]"),
                        (lambda: setattr(z, "point_count", 1), "Zone: frame_count must be in [1, 65535]"),
                        (lambda: setattr(z, "frame_count", 1), "Zone: must have either STL or ZRB"),
                        (lambda: setattr(z, "stl", api.Stl(os.path.join(ZDIR, "0.stl"))),
                         "Zone: mode must be OCCUPANCY or VACANCY"),
                        (lambda: setattr(z, "mode", api.ZoneMode.OCCUPANCY),
                         "Zone: STL coordinate frame must be BODY or SENSOR")):
        setup()
        with pytest.raises(RuntimeError, match="^" + re.escape(text) + "$"):
            z.check_invariants()
    z.stl.coordinate_frame = api.CoordinateFrame.BODY
    z.check_invariants()


def test_emulated_zone_mon_value_errors(ob):
    api = ob.pyapi
    zs = api.ZoneSet()
    with pytest.raises(ValueError, match="^ZoneSet must have at least one zone defined$"):
        api.EmulatedZoneMon(zs)
    z = api.Zone()
    z.point_count = z.frame_count = 1
    z.mode = api.ZoneMode.OCCUPANCY
    zs.zones = {0: z}
    with pytest.raises(ValueError, match="^EmulatedZoneMon: all zones in ZoneSet must have a valid ZRB$"):
        api.EmulatedZoneMon(zs)
    # test_max_count: counted from the ZRB on construction
    z.zrb = api.Zrb(np.ones((4, 4), np.uint32), np.full((4, 4), 5, np.uint32))
    assert api.EmulatedZoneMon(zs).max_counts[0] == 16
    z.zrb = api.Zrb(np.full((4, 4), 5, np.uint32), np.ones((4, 4), np.uint32))
    assert api.EmulatedZoneMon(zs).max_counts[0] == 0


def test_stl_number_parsing(ob):
    """std::stof on the vertex tokens: one rounding to the nearest float, strtof's prefix rule, and ERANGE (overflow,
    or a nonzero number that comes out subnormal or zero) raising as std::stof throws; expected values from glibc"""
    stof = ob.pyapi._stof
    assert stof(b"1.17549435e-38") == np.float32(1.17549435e-38)
    assert stof(b"3.4028235e38") == np.finfo(np.float32).max
    assert stof(b"1.2.3") == np.float32(1.2) and stof(b"-.5") == np.float32(-0.5)
    assert stof(b"0") == 0 and np.signbit(stof(b"-0")) and stof(b"0.0e-99") == 0
    # a decimal just above the midpoint between 1 and the next float: a double would round it onto the midpoint
    assert stof(b"1.00000005960464477539062500000000001") == np.nextafter(np.float32(1), np.float32(2))
    for bad in (b"1e-38", b"1.1754942e-38", b"1e-50", b"3.4028236e38", b"."):
        with pytest.raises(ValueError):
            stof(bad)
