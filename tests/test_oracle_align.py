"""CPU tests of the cloud-to-cloud ICP oracle (oracle/orc_align.c): the reference's known answers, the grid's tie
and overflow rules, median_abs, the SVD-based rotation, PoseV::exp, the early returns and the error texts; and that
the Python layer raises the reference's texts in its order before any device work."""
import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import align as oa

INT64_MIN = -(1 << 63)


def test_reference_known_answers():
    src = np.array([[x, y, z] for x in (-1.0, 0.0, 1.0) for y in (-1.0, 0.0, 1.0) for z in (-1.0, 0.0, 1.0)])
    t = np.array([0.1, -0.05, 0.025])
    m, it = oa.point_to_point_align(src, np.ascontiguousarray(src + t), max_corr_dist=0.5)
    np.testing.assert_allclose(m[:3, :3], np.eye(3), atol=1e-10)
    np.testing.assert_allclose(m[:3, 3], t, atol=1e-10)
    assert it >= 1
    s = np.array([[x, y, 0.0] for x in range(5) for y in range(5)], np.float64)
    tg = s.copy()
    tg[:, 2] = 0.2
    n = np.tile([0.0, 0.0, 1.0], (25, 1))
    m, it = oa.point_to_plane_align(s, tg, n, n, max_corr_dist=0.5)
    np.testing.assert_allclose(m[:3, :3], np.eye(3), atol=1e-10)
    np.testing.assert_allclose(m[:3, 3], [0.0, 0.0, 0.2], atol=1e-9)


def test_nearest_ties_go_to_the_earlier_cell_then_the_lower_row():
    # (0, 0.5, 0.5) is 0.5 from rows 0 and 1, in cells (-1, 0, 0) and (0, 0, 0): dx = -1 comes first
    tgt = np.array([[0.5, 0.5, 0.5], [-0.5, 0.5, 0.5]])
    assert list(oa.cloud_nearest(tgt, np.array([[0.0, 0.5, 0.5]]), 1.0, 1.0)) == [1]
    # equal rows in one cell: the lower index
    tgt = np.array([[5.0, 5.0, 5.0], [0.25, 0.5, 0.5], [0.25, 0.5, 0.5]])
    assert list(oa.cloud_nearest(tgt, np.array([[0.3, 0.5, 0.5]]), 1.0, 1.0)) == [1]
    # the same distance in (0, 0, -1) and (0, 0, 1): dz = -1 first
    tgt = np.array([[0.5, 0.5, 1.5], [0.5, 0.5, -0.5]])
    assert list(oa.cloud_nearest(tgt, np.array([[0.5, 0.5, 0.5]]), 1.0, 1.5)) == [1]
    # strictly smaller only: a distance equal to max_dist_sq is no match
    assert list(oa.cloud_nearest(tgt, np.array([[0.5, 0.5, 0.5]]), 1.0, 1.0)) == [-1]


def test_cells_overflow_to_int64_min_and_neighbours_wrap():
    assert oa.cell_coord(1e300, 1.0) == INT64_MIN
    assert oa.cell_coord(-1e300, 1.0) == INT64_MIN
    assert oa.cell_coord(np.nan, 1.0) == INT64_MIN
    assert oa.cell_coord(-0.5, 1.0) == -1 and oa.cell_coord(2.5, 2.0) == 5
    # +-1e300 rows share cell INT64_MIN; a query there visits that cell (and its wrapped neighbours INT64_MAX and
    # INT64_MIN + 1) and finds the row at distance 0; the other one is inf away
    tgt = np.array([[1e300, 0.0, 0.0], [-1e300, 0.0, 0.0], [0.1, 0.0, 0.0]])
    q = np.array([[1e300, 0.0, 0.0], [-1e300, 0.0, 0.0], [0.0, 0.0, 0.0]])
    assert list(oa.cloud_nearest(tgt, q, 1.0, 1.0)) == [0, 1, 2]
    # NaN rows are left out of the grid, a NaN query finds nothing
    tgt = np.array([[np.nan, 0.0, 0.0], [0.1, 0.0, 0.0]])
    assert list(oa.cloud_nearest(tgt, np.array([[0.0, 0.0, 0.0], [np.nan, 0.0, 0.0]]), 1.0, 1.0)) == [1, -1]


def test_median_abs_matches_numpy():
    rs = np.random.default_rng(0)
    for n in (1, 2, 7, 8, 1001, 1000):
        v = rs.normal(size=n)
        assert oa.median_abs(v) == np.median(np.abs(v))
    assert oa.median_abs(np.array([])) == 0.0


def kabsch(x, q, w):
    cx, cq = (w[:, None] * x).sum(0) / w.sum(), (w[:, None] * q).sum(0) / w.sum()
    h = ((x - cx) * w[:, None]).T @ (q - cq)
    u, _, vt = np.linalg.svd(h)
    d = np.sign(np.linalg.det(vt.T @ u.T))
    return vt.T @ np.diag([1.0, 1.0, d]) @ u.T


def test_svd_rotation_matches_numpy_kabsch():
    rs = np.random.default_rng(1)
    from scipy.spatial.transform import Rotation
    for k in range(50):
        x = rs.normal(size=(40, 3))
        r = Rotation.from_rotvec(rs.normal(size=3)).as_matrix()
        q = x @ r.T + rs.normal(0, 0.01, x.shape)
        w = rs.uniform(0.5, 1.0, 40)
        cx, cq = (w[:, None] * x).sum(0) / w.sum(), (w[:, None] * q).sum(0) / w.sum()
        cov = ((x - cx) * w[:, None]).T @ (q - cq)
        u, s, v, info = oa.svd3(cov)
        assert info == 0 and np.all(np.diff(s) <= 0)
        np.testing.assert_allclose(u @ np.diag(s) @ v.T, cov, atol=1e-12)
        rr = v @ u.T
        if np.linalg.det(rr) < 0:
            v[:, 2] *= -1
            rr = v @ u.T
        np.testing.assert_allclose(rr, kabsch(x, q, w), atol=1e-12)
    assert oa.svd3(np.full((3, 3), np.nan))[3] == 1
    u, s, v, info = oa.svd3(np.zeros((3, 3)))
    assert info == 0 and np.array_equal(s, np.zeros(3)) and np.array_equal(u, np.eye(3))


def twist(v):
    w, t = v[:3], v[3:]
    m = np.zeros((4, 4))
    m[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
    m[:3, 3] = t
    return m


@pytest.mark.parametrize("scale", [1.0, 1e-3, 1e-9, 1e-17, 0.0])
def test_posev_exp_matches_expm(scale):
    from scipy.linalg import expm
    rs = np.random.default_rng(int(-np.log10(scale)) if scale else 99)
    v = np.concatenate([rs.normal(size=3) * scale, rs.normal(size=3)])
    got = oa.posev_exp(v)
    np.testing.assert_allclose(got, expm(twist(v)), atol=1e-12 if scale >= 1e-3 else 1e-8)
    if scale < np.sqrt(np.finfo(float).eps):  # small-angle branch: I + skew(w)
        np.testing.assert_array_equal(got[:3, :3], np.eye(3) + twist(v)[:3, :3])
    if scale < np.finfo(float).eps:  # vee is the identity
        np.testing.assert_array_equal(got[:3, 3], v[3:])


def test_ldlt_reports_numerical_issue():
    a = np.diag([4.0, 0.0, 1.0, 0.0, 2.0, 3.0])
    x, info = oa.ldlt6(a, np.ones(6))
    assert info == 0  # zero pivots after the non-zero ones: Success, zeros in the pseudo-inverse
    np.testing.assert_array_equal(x, [0.25, 0.0, 1.0, 0.0, 0.5, 1.0 / 3.0])
    a = np.zeros((6, 6))
    assert oa.ldlt6(a, np.ones(6))[1] == 0  # an all-zero matrix: Success
    a = np.diag([0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    a[5, 0] = 1.0  # a column below a zero pivot that is not zero
    assert oa.ldlt6(a, np.ones(6))[1] == 1
    rs = np.random.default_rng(3)
    m = rs.normal(size=(6, 6))
    spd = m @ m.T + np.eye(6)
    x, info = oa.ldlt6(spd, np.arange(6.0))
    assert info == 0
    np.testing.assert_allclose(x, np.linalg.solve(spd, np.arange(6.0)), rtol=1e-10)


def test_small_clouds_and_no_correspondences_return_the_guess():
    rs = np.random.default_rng(4)
    g = np.eye(4)
    g[:3, 3] = [1.0 / 3.0, 2.0 / 7.0, np.pi]
    few, many = rs.normal(size=(19, 3)), rs.normal(size=(100, 3))
    for s, t in ((few, many), (many, few)):
        m, it = oa.point_to_point_align(s, t, g)
        assert np.array_equal(m, g) and it == 0
        m, it = oa.point_to_plane_align(s, t, s, t, g)
        assert np.array_equal(m, g) and it == 0
    # non-finite rows count towards the 20
    nan = np.full((20, 3), np.nan)
    m, it = oa.point_to_point_align(nan, many, g)
    assert np.array_equal(m, g) and it == 0
    # 20+ rows but no correspondence at the first iteration
    m, it = oa.point_to_point_align(many, many + 50.0, g)
    assert np.array_equal(m, g) and it == 0
    m, it = oa.point_to_plane_align(many, many + 50.0, many, many, g)
    assert np.array_equal(m, g) and it == 0


def test_error_texts_in_the_reference_order():
    s = np.zeros((25, 3))
    with pytest.raises(ValueError, match="max_corr_dist must be finite and greater than zero"):
        oa.point_to_point_align(s, s, None, np.nan)
    with pytest.raises(ValueError, match="max_corr_dist must be finite and greater than zero"):
        oa.point_to_plane_align(s, s, s[:2], s[:3], None, -1.0, 500.0)
    with pytest.raises(ValueError, match=r"max_normal_angle_deg must be finite and in \[0, 180\]"):
        oa.point_to_plane_align(s, s, s[:2], s[:3], None, 0.25, 180.5)
    with pytest.raises(ValueError, match="source_points and source_normals must have the same number of rows"):
        oa.point_to_plane_align(s, s, s[:2], s[:3], None, 0.25, 180.0)
    with pytest.raises(ValueError, match="target_points and target_normals must have the same number of rows"):
        oa.point_to_plane_align(s, s, s, s[:3], None, 0.25, 0.0)
    # the checks come before the 20-row early return
    with pytest.raises(ValueError, match="max_corr_dist"):
        oa.point_to_point_align(s[:3], s[:3], None, 0.0)


def test_python_api_raises_the_reference_texts_without_a_device():
    ob = graft.load_package()
    api = ob.pyapi
    s = np.zeros((5, 3))
    with pytest.raises(ValueError, match="max_corr_dist must be finite and greater than zero"):
        api.point_to_point_align(s, s, max_corr_dist=0.0)
    with pytest.raises(ValueError, match="max_corr_dist must be finite and greater than zero"):
        api.point_to_plane_align(s, s, s[:2], s[:3], max_corr_dist=np.inf, max_normal_angle_deg=-1.0)
    with pytest.raises(ValueError, match=r"max_normal_angle_deg must be finite and in \[0, 180\]"):
        api.point_to_plane_align(s, s, s[:2], s[:3], max_normal_angle_deg=np.nan)
    with pytest.raises(ValueError, match="source_points and source_normals must have the same number of rows"):
        api.point_to_plane_align(s, s, s[:2], s[:3])
    with pytest.raises(ValueError, match="target_points and target_normals must have the same number of rows"):
        api.point_to_plane_align(s, s, s, s[:3])


def test_abi_struct_sizes_match_the_ctypes_mirror():
    import ctypes
    ob = graft.load_package()
    capi = ob._capi
    for name, cls in [("ob_cloud_align_io", capi.CloudAlignIO), ("ob_cloud_nearest_io", capi.CloudNearestIO)]:
        assert capi.lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name
