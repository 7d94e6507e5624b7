"""CPU tests of the frame-to-map registration oracle (oracle/orc_icp.c): the reference's known answers
(tests/voxel_hashmap_test.cpp, python/tests/test_registration.py), the deterministic-reduce tree, SE3::exp and the LDLT
solve.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import expm

import __graft_entry__ as graft
from oracle import icp as oi


@pytest.fixture(scope="module", autouse=True)
def _built():
    oi.build()


def _map(points, vs=1.0, max_distance=100.0, max_pts=20):
    m = oi.VoxelHashMap3d(vs, max_distance, max_pts)
    if len(points):
        m.add_points(np.asarray(points, np.float64))
    return m


# ---- VoxelHashMap3d::get_closest_neighbor (voxel_hashmap_test.cpp) ----
def test_closest_on_empty_map_returns_sentinel():
    nb, d2 = _map([]).get_closest_neighbor([0.3, 0.2, 0.1])
    assert np.array_equal(nb, [0, 0, 0]) and d2 == oi.DBL_MAX
    nb, d2 = _map([]).get_closest_neighbor([0.3, 0.2, 0.1], 4.0)
    assert d2 == 4.0


def test_closest_exact_same_and_adjacent_voxel():
    m = _map([[0.5, 0.5, 0.5], [1.5, 0.5, 0.5]])
    nb, d2 = m.get_closest_neighbor([0.5, 0.5, 0.5])
    assert np.array_equal(nb, [0.5, 0.5, 0.5]) and d2 == 0.0
    nb, d2 = m.get_closest_neighbor([0.4, 0.5, 0.5])
    assert np.array_equal(nb, [0.5, 0.5, 0.5]) and d2 == pytest.approx(0.01)
    nb, d2 = m.get_closest_neighbor([1.2, 0.5, 0.5])           # the neighbour voxel holds the closer point
    assert np.array_equal(nb, [1.5, 0.5, 0.5]) and d2 == pytest.approx(0.09)


def test_closest_ties_first_in_shift_order_wins():
    # equal distances in the query's own voxel and its -x neighbour: the own voxel (shift (0,0,0)) is visited first
    m = _map([[1.25, 0.5, 0.5], [0.75, 0.5, 0.5]])
    nb, d2 = m.get_closest_neighbor([1.0, 0.5, 0.5])
    assert np.array_equal(nb, [1.25, 0.5, 0.5]) and d2 == 0.0625
    # empty own voxel, equal distances in +x and -x: shift (1,0,0) precedes (-1,0,0)
    m = _map([[-0.25, 0.5, 0.5], [1.25, 0.5, 0.5]])
    nb, d2 = m.get_closest_neighbor([0.5, 0.5, 0.5])
    assert np.array_equal(nb, [1.25, 0.5, 0.5]) and d2 == 0.5625


def test_closest_bound_prunes_all_or_allows_close():
    m = _map([[0.5, 0.5, 0.5]])
    nb, d2 = m.get_closest_neighbor([0.9, 0.5, 0.5], 0.01)
    assert np.array_equal(nb, [0, 0, 0]) and d2 == 0.01
    nb, d2 = m.get_closest_neighbor([0.9, 0.5, 0.5], 1.0)
    assert np.array_equal(nb, [0.5, 0.5, 0.5]) and d2 == pytest.approx(0.16)


def test_closest_negative_coordinates():
    m = _map([[-0.5, -0.5, -0.5], [-1.5, -0.5, -0.5]])
    nb, d2 = m.get_closest_neighbor([-1.1, -0.5, -0.5])
    assert np.array_equal(nb, [-1.5, -0.5, -0.5]) and d2 == pytest.approx(0.16)


@pytest.mark.parametrize("bound", [oi.DBL_MAX, 0.3])
def test_closest_agrees_with_brute_force_over_the_27_voxels(bound):
    rs = np.random.default_rng(3)
    pts = rs.random((400, 3)) * 6 - 3
    m = _map(pts, vs=1.0, max_pts=1000)
    stored = m.point_cloud()
    assert len(stored) == len(pts)      # resolution 1/1000: nothing rejected here
    for q in rs.random((200, 3)) * 6 - 3:
        nb, d2 = m.get_closest_neighbor(q, bound)
        vq = np.floor(q)
        near = stored[np.all(np.abs(np.floor(stored) - vq) <= 1, axis=1)]
        dd = ((near - q) ** 2).sum(1) if len(near) else np.empty(0)
        if len(dd) and dd.min() < bound:
            assert d2 == pytest.approx(dd.min(), rel=1e-12, abs=1e-15)
        else:
            assert d2 == bound and np.array_equal(nb, [0, 0, 0])


def test_constructor_errors_in_reference_order():
    for args, msg in [((0.5, 10.0, 0), "max_points_per_voxel"), ((0.0, 10.0, 0), "max_points_per_voxel"),
                      ((0.0, 10.0, 1), "voxel_size"), ((0.5, 0.0, 1), "max_distance"), ((-1, -1, 1), "voxel_size")]:
        with pytest.raises(ValueError, match=msg):
            oi.VoxelHashMap3d(*args)


def test_first_n_gate_and_cull():
    m = _map([[0.1, 0.1, 0.1], [0.11, 0.1, 0.1], [0.9, 0.9, 0.9]], vs=1.0, max_pts=2, max_distance=1.0)
    # resolution^2 = 1/2: the second point is rejected, the third kept
    assert np.array_equal(m.point_cloud(), [[0.1, 0.1, 0.1], [0.9, 0.9, 0.9]])
    m.add_points(np.array([[5.5, 0.5, 0.5], [-3.5, 0.5, 0.5]]))
    assert oi.cull_threshold(1.0, 1.0) == 4          # (ceil(1) + 1)^2
    ext = m.extract_voxels_far_from_location([0.0, 0.0, 0.0])   # |dv|^2 = 25 and 16 >= 4
    assert np.array_equal(ext, [[5.5, 0.5, 0.5], [-3.5, 0.5, 0.5]])
    assert m.size() == (1, 2)


def test_cull_threshold_wraps_like_int32():
    # ceil(5e9) does not fit an int: cvttsd2si gives INT32_MIN, + 1 and the square wrap
    d = (2**31 + 1) % 2**32
    sq = (d * d) % 2**32
    want = sq - 2**32 if sq >= 2**31 else sq
    assert oi.cull_threshold(5e9, 1.0) == want


# ---- ICPRegistration (python/tests/test_registration.py) ----
def test_icp_identity_on_empty_map():
    pose, it = oi.align_points_to_map(np.array([[0.0, 0, 0], [1, 0, 0]]), _map([], vs=0.5, max_distance=10.0), 1.0,
                                      0.1, 5)
    assert it == 0 and np.array_equal(pose, np.eye(4))


def test_icp_recovers_the_shifted_four_point_map():
    pts = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    m = _map(pts, vs=0.5, max_distance=10.0)
    shifted = pts + np.array([0.05, 0.02, -0.01])
    pose, it = oi.align_points_to_map(shifted, m, 0.5, 0.1, 20)
    rec = (pose[:3, :3] @ shifted.T).T + pose[:3, 3]
    np.testing.assert_allclose(rec, pts, atol=0.05)
    assert 1 <= it <= 20


def test_icp_without_correspondences_is_the_identity():
    m = _map([[0.0, 0, 0]], vs=0.5)
    pose, it = oi.align_points_to_map(np.array([[50.0, 50, 50]]), m, 0.5, 0.1, 10)
    assert it == 1 and np.array_equal(pose, np.eye(4))


def test_adaptive_threshold_defaults_and_update():
    ob = graft.load_package()
    t = ob.pyapi.AdaptiveThreshold(max_range=100.0)
    assert t.max_range == 100.0 and t.min_motion_threshold == 0.01 and t.compute_threshold() == 2.0
    t = ob.pyapi.AdaptiveThreshold(max_range=100.0, initial_threshold=1.0)
    dev = np.eye(4)
    dev[:3, 3] = [2.0, 0.0, 0.0]
    t.update_model_deviation(dev)
    assert t.compute_threshold() > 1.0
    assert t.compute_threshold() == pytest.approx(np.sqrt((1.0 + 4.0) / 2))
    c, s = np.cos(0.1), np.sin(0.1)
    rot = np.eye(4)
    rot[:2, :2] = [[c, -s], [s, c]]
    assert ob.pyapi.AdaptiveThreshold._angle(rot[:3, :3]) == pytest.approx(0.1, rel=1e-12)


def test_registration_defaults():
    reg = graft.load_package().pyapi.ICPRegistration()
    assert reg.max_num_iterations == 50 and reg.convergence_criterion == 0.0001 and reg.max_num_threads > 0


# ---- build_linear_system in parallel_deterministic_reduce's tree ----
def _tbb_tree(src, tgt, ks):
    """Plain numpy statement: halve [b, e) at b + (e - b) // 2 while it holds more than 128 pairs, sum a leaf
    sequentially from zero, parent = left + right."""
    def leaf(b, e):
        jtj, jtr = np.zeros((6, 6)), np.zeros(6)
        for i in range(b, e):
            s, r = src[i], src[i] - tgt[i]
            w = (ks * ks) / ((ks + ((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2])) ** 2)
            wsx, wsy, wsz = w * s[0], w * s[1], w * s[2]
            jtj[0, 0] += w; jtj[1, 1] += w; jtj[2, 2] += w
            jtj[3, 1] -= wsz; jtj[3, 2] += wsy; jtj[4, 0] += wsz; jtj[4, 2] -= wsx; jtj[5, 0] -= wsy; jtj[5, 1] += wsx
            wsx2, wsy2, wsz2 = wsx * s[0], wsy * s[1], wsz * s[2]
            jtj[3, 3] += wsy2 + wsz2; jtj[4, 3] -= wsx * s[1]; jtj[4, 4] += wsx2 + wsz2
            jtj[5, 3] -= wsx * s[2]; jtj[5, 4] -= wsy * s[2]; jtj[5, 5] += wsx2 + wsy2
            c = np.array([s[1] * r[2] - s[2] * r[1], s[2] * r[0] - s[0] * r[2], s[0] * r[1] - s[1] * r[0]])
            for k in range(3):
                jtr[k] += w * r[k]
                jtr[3 + k] += w * c[k]
        return jtj, jtr

    def rec(b, e):
        if e - b <= 128:
            return leaf(b, e)
        mid = b + (e - b) // 2
        lj, lr = rec(b, mid)
        rj, rr = rec(mid, e)
        return lj + rj, lr + rr
    return rec(0, len(src))


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000])
def test_linear_system_tree_matches_tbb_halving(n):
    rs = np.random.default_rng(n)
    src = rs.random((n, 3)) * 20 - 10
    tgt = src + rs.normal(0, 0.1, (n, 3))
    jtj, jtr = oi.build_linear_system(src, tgt, 0.3)
    wj, wr = _tbb_tree(src, tgt, 0.3)
    assert np.array_equal(jtj, wj) and np.array_equal(jtr, wr)
    assert np.array_equal(np.triu(jtj, 1), np.zeros((6, 6)))


# ---- Sophus SE3::exp and Eigen's LDLT ----
@pytest.mark.parametrize("seed", range(6))
def test_se3_exp_matches_the_matrix_exponential(seed):
    rs = np.random.default_rng(seed)
    a = rs.normal(0, [1, 1, 1, 0.5, 0.5, 0.5]) * (10.0 ** -rs.integers(0, 9))
    W = np.zeros((4, 4))
    W[:3, 3] = a[:3]
    w = a[3:]
    W[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
    np.testing.assert_allclose(oi.se3_exp(a), expm(W), rtol=0, atol=1e-13)


def test_se3_exp_small_angle_branch():
    a = np.array([0.1, 0.2, 0.3, 1e-17, 0, 0])
    m = oi.se3_exp(a)
    np.testing.assert_allclose(m[:3, 3], a[:3], atol=1e-16)
    assert np.array_equal(oi.se3_exp(np.zeros(6)), np.eye(4))


@pytest.mark.parametrize("seed", range(8))
def test_ldlt_solve_matches_numpy_on_spd_systems(seed):
    rs = np.random.default_rng(seed)
    a = rs.normal(size=(6, 6))
    a = a @ a.T + 0.1 * np.eye(6) * (seed + 1)
    b = rs.normal(size=6)
    np.testing.assert_allclose(oi.ldlt_solve(np.tril(a), b), np.linalg.solve(a, b), rtol=1e-9, atol=1e-12)


def test_ldlt_zero_system_gives_zero_step():
    assert np.array_equal(oi.ldlt_solve(np.zeros((6, 6)), np.zeros(6)), np.zeros(6))
    assert np.array_equal(oi.ldlt_solve(np.zeros((6, 6)), np.ones(6)), np.zeros(6))


# ---- C ABI ----
def test_new_structs_in_abi_sizeof_match_ctypes():
    ob = graft.load_package()
    capi = ob._capi
    for name, cls in [("ob_point_rows", capi.PointRows), ("ob_voxel_map_cull_io", capi.VoxelMapCullIO),
                      ("ob_voxel_query_io", capi.VoxelQueryIO), ("ob_icp_io", capi.IcpIO),
                      ("ob_icp_system_io", capi.IcpSystemIO)]:
        assert capi.lib.ob_abi_sizeof(name.encode()) == C.sizeof(cls), name


def test_map_constructor_errors_and_no_device_through_the_abi():
    ob = graft.load_package()
    for args, msg in [((0.5, 10.0, 0), "max_points_per_voxel must be greater than 0"),
                      ((0.0, 10.0, 1), "voxel_size must be greater than 0"),
                      ((0.5, -1.0, 1), "max_distance must be greater than 0")]:
        with pytest.raises(ValueError, match=msg):
            ob.pyapi.VoxelHashMap3d(*args)
    if ob.device_count() == 0:
        with pytest.raises(ob._capi.OusterB200Error, match="status 4"):
            ob.pyapi.VoxelHashMap3d(0.5)
    for fam in ("voxel_map", "icp"):
        assert ob.kernel_launch_count(fam) >= 0
