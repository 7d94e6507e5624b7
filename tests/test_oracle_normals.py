"""Pins the normals oracle (oracle/orc_normals.c) to the reference's own known answers
(python/tests/test_normals.py:362-442, regression values written into the reference's test) and to
geometric properties (unit length, planar scenes as test_normals_cube_boundaries checks them)."""
import numpy as np
import pytest

from oracle import oracle as orc


def test_reference_known_answers_single_and_dual():
    # python/tests/test_normals.py:362-401 (test_normals)
    xyz = np.array([[[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]], [[0.0, 1.0, 0.0], [1.0, 1.0, 0.0]]])
    rng = np.array([[0.0, 1.0], [1.0, 1.0]], np.uint32)
    org = np.zeros((2, 3))
    want = np.array([[[0.0, 0.0, 0.0], [-1.0, 0.0, 0.0]], [[0.0, -1.0, 0.0], [-0.70710678, -0.70710678, 0.0]]])
    got = orc.normals(xyz, rng, sensor_origins_xyz=org, pixel_search_range=1, min_angle_of_incidence_rad=0.1,
                      target_distance_m=100)
    assert np.allclose(got, want)
    got1, got2 = orc.normals(xyz, rng, xyz, rng, org, 1, 0.1, 100)
    assert np.allclose(got1, want)


def test_reference_known_answers_isolated_pixel():
    # python/tests/test_normals.py:404-442 (test_normals_2)
    xyz = np.array([[[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]], [[0.0, 0.0, 0.0], [0.0, 0.0, 0.0]]])
    rng = np.array([[0.0, 1.0], [0.0, 0.0]], np.uint32)
    org = np.zeros((2, 3))
    want = np.array([[[0.0, 0.0, 0.0], [-1.0, 0.0, 0.0]], [[0.0, 0.0, 0.0], [0, 0.0, 0.0]]])
    assert np.allclose(orc.normals(xyz, rng, sensor_origins_xyz=org, pixel_search_range=1,
                                   min_angle_of_incidence_rad=0.1, target_distance_m=100), want)
    got1, _ = orc.normals(xyz, rng, xyz, rng, org, 1, 0.1, 100)
    assert np.allclose(got1, want)


def test_reference_error_texts():
    # python/tests/test_normals.py:212-359
    xyz = np.zeros((2, 2, 3))
    rng = np.ones((2, 2), np.uint32)
    with pytest.raises(RuntimeError, match="target_distance_m must be positive"):
        orc.normals(xyz, rng, sensor_origins_xyz=np.zeros((2, 3)), target_distance_m=-100)
    with pytest.raises(RuntimeError, match="min_angle_of_incidence_rad must be positive"):
        orc.normals(xyz, rng, sensor_origins_xyz=np.zeros((2, 3)), min_angle_of_incidence_rad=-0.1)
    with pytest.raises(RuntimeError, match="sensor_origins size must match image width"):
        orc.normals(xyz, rng, sensor_origins_xyz=np.zeros((0, 3)))
    with pytest.raises(RuntimeError, match="xyz dimensions mismatch"):
        orc.normals(xyz, np.ones((1, 2), np.uint32), sensor_origins_xyz=np.zeros((2, 3)))


def room_scene(h=64, w=512, half=40000.0, seed=0):
    """Sensor at the origin of a cube room (walls at +-half mm; 40 m keeps the 1 mm range quantisation below 0.2 deg): destaggered XYZ (metres) and range (mm)
    of a spinning lidar with +-22.5 deg vertical field of view."""
    alt = np.deg2rad(np.linspace(22.5, -22.5, h))[:, None]
    az = (2 * np.pi * (1 - np.arange(w) / w))[None, :]
    d = np.stack([np.cos(az) * np.cos(alt), np.sin(az) * np.cos(alt), np.sin(alt) * np.ones_like(az)], -1)
    t = half / np.max(np.abs(d), axis=-1)           # distance to the nearest wall along the beam
    rng = np.round(t).astype(np.uint32)
    xyz = d * rng[..., None] * 0.001
    return xyz, rng, d


def test_planar_room_normals_point_inwards_and_are_unit():
    xyz, rng, d = room_scene()
    n = orc.normals(xyz, rng, sensor_origins_xyz=np.zeros((xyz.shape[1], 3)))
    norms = np.linalg.norm(n, axis=-1)
    assert np.all(norms[rng > 0] > 0)
    assert np.allclose(norms[rng > 0], 1.0, atol=1e-9)
    # away from the wall edges the normal is the inward wall normal (test_normals_cube_boundaries: 0.5 deg)
    axis = np.argmax(np.abs(d), axis=-1)
    expected = np.zeros_like(d)
    np.put_along_axis(expected, axis[..., None], -np.sign(np.take_along_axis(d, axis[..., None], -1)), -1)
    cosang = np.sum(n * expected, -1)
    sorted_abs = np.sort(np.abs(d), axis=-1)
    interior = sorted_abs[..., 2] - sorted_abs[..., 1] > 0.05      # not next to an edge of the cube
    assert np.mean(cosang[interior] > np.cos(np.deg2rad(0.5))) > 0.99


def test_dual_return_shares_the_vertical_subtent():
    xyz, rng, _ = room_scene(32, 128)
    rs = np.random.default_rng(3)
    rng2 = np.where(rs.random(rng.shape) < 0.3, rng + 700, 0).astype(np.uint32)
    xyz2 = xyz * (rng2 / np.maximum(rng, 1))[..., None]
    org = np.zeros((128, 3))
    n1, n2 = orc.normals(xyz, rng, xyz2, rng2, org)
    sub = orc.normals_vertical_subtent(xyz, rng, org)
    a1, a2 = orc.normals(xyz, rng, xyz2, rng2, org, vertical_subtent=sub)
    assert np.array_equal(n1, a1) and np.array_equal(n2, a2)
    assert np.all(n2[rng2 == 0] == 0)


# ------------------------------------------------------------------------------------------------
# Scenes built to reach one branch of compute_unit_normals each, with a float64 expectation beside
# the oracle's answer.  tests/test_gpu_normals_edges.py runs the same scenes on the GPU.
# ------------------------------------------------------------------------------------------------
def grid_dirs(alt, az):
    """Unit beam directions; rows are altitudes (top row first), columns azimuths (decreasing with the
    column, as a spinning lidar's destaggered image)."""
    alt = np.asarray(alt, np.float64)[:, None]
    az = np.asarray(az, np.float64)[None, :]
    return np.stack([np.cos(az) * np.cos(alt), np.sin(az) * np.cos(alt), np.sin(alt) * np.ones_like(az)], -1)


def dot_rows(a, b):
    """(a0 b0 + a1 b1) + a2 b2, the summation order of the reference's 3-vector dot."""
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def beams_of(xyz, org):
    """normals.cpp:111-129 in numpy: (xyz - origin of the column) / its norm, zero for a zero vector."""
    dvec = xyz - org[None]
    mag = np.sqrt(dot_rows(dvec, dvec))
    with np.errstate(invalid="ignore", divide="ignore"):
        b = dvec / mag[..., None]
    b[~(mag > 0)] = 0.0
    return b


def wall_scene(h=12, w=24, wall_m=8.0, a=0.004):
    """A wall at x = wall_m seen over a small grid (a radians between rows and between columns)."""
    d = grid_dirs(a * ((h - 1) / 2 - np.arange(h)), -a * (np.arange(w) - (w - 1) / 2))
    t = wall_m / d[..., 0]
    return d * t[..., None], np.round(t * 1000).astype(np.uint32), d


def _put(xyz, rng, d, u, v, t_m):
    xyz[u, v] = d[u, v] * t_m
    rng[u, v] = np.uint32(round(t_m * 1000))


def _isolated_pixel_case(neighbours):
    """Pixel (5, 10) at 5 m in front of the 8 m wall; its four radius-1 neighbours are the wall, the
    wall with range cr + 500 or cr + 499, or invalid."""
    xyz, rng, d = wall_scene()
    _put(xyz, rng, d, 5, 10, 5.0)
    cr = int(rng[5, 10])
    for u, v in ((4, 10), (6, 10), (5, 9), (5, 11)):
        if neighbours == "invalid":
            rng[u, v] = 0
        elif neighbours != "wall":
            rng[u, v] = cr + neighbours
    org = np.zeros((xyz.shape[1], 3))
    beam = beams_of(xyz, org)[5, 10]

    def check(n):
        if neighbours == 499:                           # one neighbour 499 mm behind: not thin, not case A
            assert not np.array_equal(n[5, 10], -beam)
        else:                                           # case A: the beam itself, exactly
            assert np.array_equal(n[5, 10], -beam)
    return dict(xyz=xyz, rng=rng, org=org, kw={}, check=check)


def _pole_case():
    """Case B-vertical: a one-column pole (x = 5 m) 3 m in front of the wall: its vertical neighbours lie
    on the pole, its horizontal ones are >= 500 mm farther.  The pole is parallel to z, so the normal is
    minus the horizontal part of the beam."""
    xyz, rng, d = wall_scene()
    for u in range(xyz.shape[0]):
        _put(xyz, rng, d, u, 10, 5.0 / d[u, 10, 0])
    org = np.zeros((xyz.shape[1], 3))

    def check(n):
        b = beams_of(xyz, org)[:, 10]
        flat = b * np.array([1.0, 1.0, 0.0])
        want = -flat / np.linalg.norm(flat, axis=-1, keepdims=True)
        assert np.allclose(n[:, 10], want, rtol=0, atol=1e-9)
    return dict(xyz=xyz, rng=rng, org=org, kw={}, check=check)


def _check_perpendicular(n, beam, diff):
    """n is the unit vector in span(beam, diff) perpendicular to diff, on the sensor's side."""
    scale = np.linalg.norm(diff)
    assert abs(np.linalg.norm(n) - 1.0) < 1e-12
    assert abs(n @ diff) <= 1e-12 * scale
    assert abs(np.linalg.det(np.stack([n, beam, diff]))) <= 1e-12 * scale
    assert n @ beam < 0


def _strip_case():
    """Case B-horizontal: a one-row strip (row 6, x = 5 m) in front of the wall; the neighbour chosen is
    the left or right one whose squared distance is nearer the target's (left wins ties)."""
    xyz, rng, d = wall_scene()
    h, w = rng.shape
    for v in range(w):
        _put(xyz, rng, d, 6, v, 5.0 / d[6, v, 0])
    org = np.zeros((w, 3))

    def check(n):
        b = beams_of(xyz, org)
        t_sq = orc.DEFAULT_TARGET_DISTANCE_METER ** 2
        for v in range(w):
            dl, dr = xyz[6, (v - 1) % w] - xyz[6, v], xyz[6, (v + 1) % w] - xyz[6, v]
            pick = dr if abs(dot_rows(dr, dr) - t_sq) < abs(dot_rows(dl, dl) - t_sq) else dl
            _check_perpendicular(n[6, v], b[6, v], pick)
    return dict(xyz=xyz, rng=rng, org=org, kw={}, check=check)


def _degenerate_case(kind):
    """Pixel (5, 10) at 5 m whose only valid radius-1 neighbour is the one above it:
    on_beam    -- 300 mm farther along the pixel's own beam: the beam has no component perpendicular to
                  it, so a valid pixel gets the zero normal;
    near_dup   -- 1 nm away: accepted (> 0 at the last radius), but its squared length is below epsilon;
    duplicate  -- the same point: a squared distance of 0 is never accepted, so the pixel is case A."""
    xyz, rng, d = wall_scene()
    _put(xyz, rng, d, 5, 10, 5.0)
    for u, v in ((6, 10), (5, 9), (5, 11)):
        rng[u, v] = 0
    if kind == "on_beam":
        xyz[4, 10] = d[5, 10] * 5.3
        rng[4, 10] = 5300
    else:
        xyz[4, 10] = xyz[5, 10] + (np.array([1e-9, 0.0, 0.0]) if kind == "near_dup" else 0.0)
        rng[4, 10] = rng[5, 10]
    org = np.zeros((xyz.shape[1], 3))
    beam = beams_of(xyz, org)[5, 10]

    def check(n):
        assert rng[5, 10] > 0
        assert np.array_equal(n[5, 10], -beam if kind == "duplicate" else np.zeros(3))
    return dict(xyz=xyz, rng=rng, org=org, kw={}, check=check)


def _aoi_case(aoi):
    """Pixel (5, 10) at 10 m with the vertical subtent fixed at 0.01 rad, so the vertical gate is
    (10 m * 0.01) / tan(max(aoi, 1e-6)).  Its one neighbour (above) is 2 m away at 45 deg to the beam:
    inside the gate at 1 deg (5.73 m) and at 1e-9 (clamped to 1e-6), outside it at 10 deg (0.567 m)."""
    xyz, rng, d = wall_scene()
    _put(xyz, rng, d, 5, 10, 10.0)
    for u, v in ((6, 10), (5, 9), (5, 11)):
        rng[u, v] = 0
    beam = d[5, 10] / np.linalg.norm(d[5, 10])
    perp = np.cross(beam, [0.0, 0.0, 1.0])
    perp /= np.linalg.norm(perp)
    xyz[4, 10] = xyz[5, 10] + np.sqrt(2.0) * (beam + perp)
    rng[4, 10] = rng[5, 10]
    org = np.zeros((xyz.shape[1], 3))
    b = beams_of(xyz, org)[5, 10]

    def check(n):
        if aoi == np.deg2rad(10.0):                     # gated out: no neighbour, case A
            assert np.array_equal(n[5, 10], -b)
        else:                                           # case B-vertical: (perp - beam) / sqrt(2)
            assert np.allclose(n[5, 10], (perp - beam) / np.sqrt(2.0), rtol=0, atol=1e-9)
    return dict(xyz=xyz, rng=rng, org=org, kw=dict(min_angle_of_incidence_rad=aoi, vertical_subtent=0.01),
                check=check)


def plane_scene(dist, h=16, w=24, a=0.004):
    """A tilted plane n.x = -dist (n the unit normal facing the sensor), every point exactly t * dir.
    Angular gaps alternate a and 3a along both axes, and the target distance is dist * a, so each
    pixel's chosen neighbour is the one across the small gap: above it on odd rows, to its left on odd
    columns.  All four flip combinations of case C occur."""
    gaps = lambda k: np.where(np.arange(k - 1) % 2 == 0, a, 3 * a)
    alt = 0.05 - np.concatenate([[0.0], np.cumsum(gaps(h))])
    az = 0.2 - np.concatenate([[0.0], np.cumsum(gaps(w))])
    d = grid_dirs(alt, az)
    n_face = np.array([-1.0, 0.3, -0.2]) / np.linalg.norm([-1.0, 0.3, -0.2])
    t = -dist / dot_rows(d, n_face)
    return d * t[..., None], np.round(t * 1000).astype(np.uint32), n_face, dist * a


def _plane_case(dist):
    xyz, rng, n_face, target = plane_scene(dist)
    h, w = rng.shape
    org = np.zeros((w, 3))

    def check(n):
        assert np.allclose(n, np.broadcast_to(n_face, n.shape), rtol=0, atol=1e-9)
        # which side each interior pixel picks (the first candidate wins ties), all four combinations
        t_sq = target * target
        sq = lambda a_: dot_rows(a_, a_)
        c = xyz[1:-1, 1:-1]
        vflip = ~(abs(sq(xyz[2:, 1:-1] - c) - t_sq) < abs(sq(xyz[:-2, 1:-1] - c) - t_sq))
        hflip = ~(abs(sq(xyz[1:-1, 2:] - c) - t_sq) < abs(sq(xyz[1:-1, :-2] - c) - t_sq))
        assert {(a_, b_) for a_, b_ in zip(vflip.ravel(), hflip.ravel())} == {(False, False), (False, True),
                                                                           (True, False), (True, True)}
    return dict(xyz=xyz, rng=rng, org=org, kw=dict(target_distance_m=target), check=check)


BRANCH_CASES = {
    "A_thin_wall": lambda: _isolated_pixel_case("wall"),
    "A_wall_500mm_behind": lambda: _isolated_pixel_case(500),
    "not_A_wall_499mm_behind": lambda: _isolated_pixel_case(499),
    "A_no_valid_neighbours": lambda: _isolated_pixel_case("invalid"),
    "B_vertical_pole": _pole_case,
    "B_horizontal_strip": _strip_case,
    "B_neighbour_on_beam": lambda: _degenerate_case("on_beam"),
    "B_neighbour_within_eps": lambda: _degenerate_case("near_dup"),
    "duplicate_never_accepted": lambda: _degenerate_case("duplicate"),
    "aoi_1deg": lambda: _aoi_case(np.deg2rad(1.0)),
    "aoi_10deg": lambda: _aoi_case(np.deg2rad(10.0)),
    "aoi_1e-9_clamped": lambda: _aoi_case(1e-9),
    "C_plane_2m": lambda: _plane_case(2.0),
    "C_plane_6m": lambda: _plane_case(6.25),
    "C_plane_30m": lambda: _plane_case(30.0),
}


@pytest.mark.parametrize("name", list(BRANCH_CASES))
def test_branch_scene_matches_float64_expectation(name):
    c = BRANCH_CASES[name]()
    c["check"](orc.normals(c["xyz"], c["rng"], sensor_origins_xyz=c["org"], **c["kw"]))


def test_aoi_below_1e6_is_clamped():
    xyz, rng, _ = room_scene(24, 96)
    org = np.zeros((96, 3))
    a = orc.normals(xyz, rng, sensor_origins_xyz=org, min_angle_of_incidence_rad=1e-9)
    assert np.array_equal(a, orc.normals(xyz, rng, sensor_origins_xyz=org, min_angle_of_incidence_rad=1e-6))


# ------------------------------------------------------------------------------------------------
# compute_vertical_subtent: candidate order mid, mid, mid-1, mid+1, ..., inward walk, fallback
# ------------------------------------------------------------------------------------------------
def subtent_scene(h, w, columns, seed=0):
    """Only the listed columns hold returns: {col: (alt_top_rad, alt_bottom_rad, holes_at_row0,
    holes_at_last_row)}; rows in between are valid, at 10 m.  Everything else has range 0."""
    xyz = np.zeros((h, w, 3))
    rng = np.zeros((h, w), np.uint32)
    az = -0.003 * (np.arange(w) - w / 2)
    for col, (a0, a1, b, e) in columns.items():
        dcol = grid_dirs(np.linspace(a0, a1, h), [az[col]])[:, 0]
        xyz[:, col] = dcol * 10.0
        rng[b:h - e, col] = 10000
    org = np.random.default_rng(seed).normal(0, 0.01, (w, 3))
    return xyz, rng, org


def expected_subtent(xyz, rng, org, col):
    """The float64 value compute_vertical_subtent returns when column `col` is the one it settles on."""
    valid = np.nonzero(rng[:, col])[0]
    bottom, top = valid[0], valid[-1]
    b = beams_of(xyz, org)
    dp = min(1.0, max(-1.0, float(dot_rows(b[top, col], b[bottom, col]))))
    return float(np.arccos(dp)) / (top - bottom)


def ulps(a, b):
    return abs(a - b) / np.spacing(max(abs(a), abs(b)))


# (W, columns, the column the search must settle on)
SUBTENT_SEARCH_CASES = {
    "mid_invalid_even_W": (10, {4: (0.3, -0.3, 0, 0), 6: (0.5, -0.5, 0, 0)}, 4),
    "mid_invalid_odd_W": (9, {3: (0.2, -0.1, 2, 1), 5: (0.5, -0.5, 0, 0)}, 3),
    "mid_single_pixel": (10, {5: (0.3, -0.3, 3, 9), 4: (0.1, -0.3, 1, 4), 6: (0.5, -0.5, 0, 0)}, 4),
    "mid_plus_one_when_mid_minus_one_empty": (11, {6: (0.4, -0.2, 5, 0), 7: (0.1, -0.1, 0, 0)}, 6),
    "holes_at_both_ends_of_mid": (12, {6: (0.25, -0.35, 4, 2), 5: (0.5, -0.5, 0, 0)}, 6),
    "second_warp_iteration": (101, {50 + 15: (0.3, -0.3, 1, 0), 50 - 16: (0.1, -0.1, 0, 1),
                                    50 + 20: (0.5, -0.5, 0, 0)}, 65),
    "beyond_32_candidates": (101, {50 + 20: (0.3, -0.3, 2, 3), 50 - 21: (0.5, -0.5, 0, 0)}, 70),
}


@pytest.mark.parametrize("name", list(SUBTENT_SEARCH_CASES))
def test_subtent_search_order_and_inward_walk(name):
    w, cols, want_col = SUBTENT_SEARCH_CASES[name]
    xyz, rng, org = subtent_scene(13, w, cols)
    got = orc.normals_vertical_subtent(xyz, rng, org)
    want = expected_subtent(xyz, rng, org, want_col)
    assert ulps(got, want) <= 8
    for col in cols:                                   # the other columns give clearly different values
        if col != want_col and np.count_nonzero(rng[:, col]) >= 2:
            assert ulps(got, expected_subtent(xyz, rng, org, col)) > 1e6


@pytest.mark.parametrize("h,valid", [(1, True), (2, False), (2, "one_row"), (5, False)])
def test_subtent_fallback_is_90_degrees_over_the_height(h, valid):
    xyz, rng, _ = room_scene(h, 16)
    if valid is False:
        rng[:] = 0
    elif valid == "one_row":
        rng[1] = 0
    got = orc.normals_vertical_subtent(xyz, rng, np.zeros((16, 3)))
    assert got == (0.5 * np.pi) / max(1, h - 1)


# ------------------------------------------------------------------------------------------------
# Dual returns whose first return has a vertical subtent of 0
# ------------------------------------------------------------------------------------------------
def dual_zero_subtent_scene(kind, h=32, w=128, seed=4):
    """Room scene whose first return's subtent is exactly 0: the first valid top/bottom pair of the
    centre column lies on one ray along +x ("parallel": the beams are equal, acos(1) = 0) or has an
    infinite coordinate ("inf": the beam is NaN, which the clamp turns into a dot product of 1).  The
    second return is an ordinary scene 700 mm behind the first."""
    rs = np.random.default_rng(seed)
    xyz, rng, d = room_scene(h, w)
    rng[rs.random(rng.shape) < 0.1] = 0
    mid = w // 2
    rng[0, mid] = rng[h - 1, mid] = 20000
    xyz = d * rng[..., None] * 0.001
    rng2 = np.where(rng > 0, rng + 700, 0).astype(np.uint32)
    xyz2 = d * rng2[..., None] * 0.001
    org = rs.normal(0, 0.05, (w, 3))
    if kind == "parallel":
        org[mid] = 0.0
        xyz[0, mid] = (20.0, 0.0, 0.0)
        xyz[h - 1, mid] = (7.5, 0.0, 0.0)
    else:
        xyz[h - 1, mid, 0] = np.inf
    return xyz, rng, xyz2, rng2, org


@pytest.mark.parametrize("kind", ["parallel", "inf"])
def test_dual_zero_subtent_second_return_derives_its_own(kind):
    x1, r1, x2, r2, org = dual_zero_subtent_scene(kind)
    assert orc.normals_vertical_subtent(x1, r1, org) == 0.0
    s2 = orc.normals_vertical_subtent(x2, r2, org)
    mid = x1.shape[1] // 2
    assert s2 > 0 and ulps(s2, expected_subtent(x2, r2, org, mid)) <= 8
    n1, n2 = orc.normals(x1, r1, x2, r2, org)
    m2, m1 = orc.normals(x2, r2, x1, r1, org)
    # the reference's second pass is the same pass as the swapped call's first: subtent of (xyz2, range2)
    assert np.array_equal(n2, m2)
    # the rule matters here: a second pass that kept the shared subtent of 0 (emulated by the smallest
    # subnormal, for which 2 pi / subtent overflows just as 2 pi / 0 does) differs on most pixels
    z1, z2 = orc.normals(x1, r1, x2, r2, org, vertical_subtent=5e-324)
    assert np.array_equal(z1, n1, equal_nan=True)
    assert np.mean(np.any(z2 != n2, axis=-1)[r2 > 0]) > 0.5
