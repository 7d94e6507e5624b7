"""Pins the voxel-downsampling oracle (oracle/orc_voxel.c) to the reference's known answers and test
properties (python/tests/test_core.py:486-510, tests/voxel_downsample_test.cpp), and checks the two
reformulations the GPU pipeline uses (tests/voxel_reference.py) against the oracle's sequential loops."""
import numpy as np
import pytest

from oracle import oracle as orc
from oracle import voxel as orv
from tests import voxel_reference as vr

INT32_MIN = -2147483648


def same_rows(a, b):
    """Row multisets equal (the reference emits in hash-map order)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])])


def test_reference_known_answer_xd_average():
    # python/tests/test_core.py:486-510 (test_voxel_downsample_xd), compared order-independently as there
    pts = np.array([[0.0, 1.0, 0.0], [0.0, 1.0, 0.0], [0.0, 2.0, 0.0], [0.0, 2.0, 0.0]])
    attrs = np.array([[10.0, 100.0], [12.0, 102.0], [20.0, 200.0], [22.0, 202.0]])
    frame = np.hstack([pts, attrs])
    got = orv.voxel_downsample_xd(frame, 0.1, 1, 1, orv.AVERAGE_POINT)
    assert same_rows(got, [[0.0, 2.0, 0.0, 21.0, 201.0], [0.0, 1.0, 0.0, 11.0, 101.0]])
    got = orv.voxel_downsample_xd(frame, 4.0, 1, 1, orv.AVERAGE_POINT)
    assert same_rows(got, [[0.0, 1.5, 0.0, 16.0, 151.0]])


# ---- properties of core::voxel_downsample, restated from tests/voxel_downsample_test.cpp ----
def test_empty_and_single_point():
    p, i = orv.voxel_downsample(np.empty((0, 3)), 1.0)
    assert p.shape == (0, 3) and i.shape == (0,)
    p, i = orv.voxel_downsample(np.array([[1.0, 2.0, 3.0]]), 1.0)
    assert np.array_equal(p, [[1.0, 2.0, 3.0]]) and np.array_equal(i, [0])


def test_points_in_distinct_voxels_all_kept_and_indices_match():
    rs = np.random.default_rng(0)
    frame = np.arange(50, dtype=np.float64)[:, None] * np.array([[1.0, 0.0, 0.0]]) + rs.random((50, 3)) * 0.1
    p, i = orv.voxel_downsample(frame, 0.5)
    assert len(p) == 50 and np.array_equal(p, frame[i]) and len(set(i.tolist())) == 50


def test_one_representative_per_voxel_from_the_input():
    rs = np.random.default_rng(1)
    frame = rs.random((3000, 3)) * 10
    p, i = orv.voxel_downsample(frame, 1.0)
    vox = vr.voxel_keys(p, 1.0)
    assert len({tuple(v) for v in vox}) == len(p) == len({tuple(v) for v in vr.voxel_keys(frame, 1.0)})
    assert np.array_equal(p, frame[i]) and len(set(i.tolist())) == len(i) and i.max() < len(frame)
    p2, i2 = orv.voxel_downsample(frame, 1.0)            # deterministic (seed 42)
    assert np.array_equal(p, p2) and np.array_equal(i, i2)


def test_does_not_always_pick_the_first_point():
    base = np.arange(200, dtype=np.float64)[:, None] * np.array([[0.01, 0.0, 0.0]])
    rs = np.random.default_rng(777)
    picked = set()
    for _ in range(20):
        frame = base[rs.permutation(200)]
        p, _ = orv.voxel_downsample(frame, 100.0)
        assert len(p) == 1
        picked.add(int(round(p[0, 0] / 0.01)))
    assert len(picked) > 1


# ---- the GPU's reformulations ----
@pytest.mark.parametrize("n", list(range(1, 40)) + [63, 64, 65, 255, 256, 257, 1000, 1023, 1024, 1025, 4096, 4097])
def test_parallel_fisher_yates_equals_the_sequential_shuffle(n):
    frame = np.zeros((n, 3))
    frame[:, 0] = np.arange(n)                            # one voxel per point: indices_out is the permutation
    _, idx = orv.voxel_downsample(frame, 0.5)
    assert np.array_equal(vr.parallel_shuffle(n), idx)


def test_jump_matrices_equal_sequential_xorshift():
    s, seq = 42, []
    for _ in range(5000):
        s = vr.xs_step(s)
        seq.append(s)
    k = np.arange(5000, dtype=np.uint64)
    assert np.array_equal(vr.xs_state_after(k + np.uint64(1)), np.array(seq, np.uint64))
    s = 42
    for _ in range(1 << 20):
        s = vr.xs_step(s)
    assert int(vr.xs_state_after(np.array([1 << 20], np.uint64))[0]) == s


@pytest.mark.parametrize("max_pts", [1, 3, 8])
def test_random_draw_index_formulation_equals_the_oracle(max_pts):
    rs = np.random.default_rng(max_pts)
    frame = np.vstack([rs.random((2000, 3)) * 4, rs.random((500, 3)) * 0.2])   # sparse voxels and a dense one
    got, idx = orv.voxel_downsample_xd(frame, 0.5, max_pts, 1, orv.RANDOM, with_indices=True)
    assert np.array_equal(vr.random_by_draw_index(frame, 0.5, max_pts), idx)
    assert np.array_equal(got, frame[idx])


def test_nan_and_huge_coordinates_share_the_int_min_voxel():
    assert orv.voxel_coord(float("nan")) == INT32_MIN
    assert orv.voxel_coord(1e300) == INT32_MIN and orv.voxel_coord(-1e300) == INT32_MIN
    assert orv.voxel_coord(float("inf")) == INT32_MIN
    assert orv.voxel_coord(2147483648.0) == INT32_MIN and orv.voxel_coord(-2147483649.0) == INT32_MIN
    assert orv.voxel_coord(2147483647.5) == 2147483647 and orv.voxel_coord(-2147483648.0) == INT32_MIN
    assert orv.voxel_coord(-0.5) == -1
    frame = np.array([[np.nan, np.nan, np.nan], [1e300, -1e300, np.inf], [0.1, 0.1, 0.1]])
    out = orv.voxel_downsample_xd(frame, 1.0, 1, 1, orv.FIRST_N_POINT)
    assert np.array_equal(out, frame[[0, 2]], equal_nan=True)
    out = orv.voxel_downsample_xd(frame, 1.0, 1, 1, orv.AVERAGE_POINT)
    assert np.isnan(out[0]).all() and np.array_equal(out[1], frame[2])
    assert np.array_equal(vr.voxel_keys(frame, 1.0)[:2], np.full((2, 3), INT32_MIN))


def test_first_n_distance_gate_and_min_points():
    frame = np.array([[0.1, 0.1, 0.1], [0.15, 0.1, 0.1], [0.9, 0.9, 0.9], [0.7, 0.7, 0.7], [3.5, 0.0, 0.0]])
    # res^2 = 1/3: the second point is too close to the first, the fourth to the third
    out, idx = orv.voxel_downsample_xd(frame, 1.0, 3, 1, orv.FIRST_N_POINT, with_indices=True)
    assert np.array_equal(idx, [0, 2, 4])
    # min_pts_threshold applies to AVERAGE_POINT only
    assert len(orv.voxel_downsample_xd(frame, 1.0, 3, 4, orv.FIRST_N_POINT)) == 3
    out = orv.voxel_downsample_xd(frame, 1.0, 1, 4, orv.AVERAGE_POINT)
    assert np.array_equal(out, [np.sum(frame[:4], axis=0) / 4.0])


def test_with_normals_averages_and_renormalises():
    pts = np.array([[0.1, 0.1, 0.1], [0.3, 0.1, 0.1], [5.2, 0.0, 0.0], [np.nan, 0, 0], [0.2, 0.2, 0.2], [7.0, 0, 0]])
    nrm = np.array([[0.0, 0.0, 2.0], [0.0, 3.0, 0.0], [1.0, 0.0, 0.0], [1.0, 0, 0], [0.0, 0.0, 0.0], [0.0, 0, 1e-13]])
    p, n = orv.voxel_downsample_with_normals(pts, nrm, 1.0)
    assert np.array_equal(p, [[(0.1 + 0.3) / 2, 0.1, 0.1], [5.2, 0.0, 0.0]])
    assert np.allclose(n, [[0.0, np.sqrt(0.5), np.sqrt(0.5)], [1.0, 0.0, 0.0]], atol=0, rtol=1e-15)
    # opposite unit normals cancel: the voxel is dropped
    p, n = orv.voxel_downsample_with_normals(np.array([[0.1, 0, 0], [0.2, 0, 0]]), np.array([[0, 0, 1.0], [0, 0, -1.0]]), 1.0)
    assert p.shape == (0, 3) and n.shape == (0, 3)


def test_error_texts_and_their_order():
    frame = np.zeros((4, 3))
    with pytest.raises(ValueError, match="^max_points_per_voxel must be greater than 0$"):
        orv.voxel_downsample_xd(frame, -1.0, 0, 1, orv.RANDOM)        # checked before voxel_size
    with pytest.raises(ValueError, match="^voxel_size must be greater than 0$"):
        orv.voxel_downsample_xd(frame, 0.0, 1, 1, orv.FIRST_N_POINT)
    with pytest.raises(ValueError, match="^voxel_downsample_xd: frame must have at least 3 columns$"):
        orv.voxel_downsample_xd(np.zeros((4, 2)), 1.0)
    with pytest.raises(ValueError, match="^voxel_downsample_xd: unknown strategy$"):
        orv.voxel_downsample_xd(frame, -1.0, 0, 1, 7)                 # the switch runs before the map is built
    with pytest.raises(ValueError, match="^voxel_downsample_3d: unknown strategy$"):
        orv.voxel_downsample_xd(frame, 1.0, 1, 1, 7, name="voxel_downsample_3d")
    with pytest.raises(ValueError, match="^voxel_downsample_with_normals expects Nx3 inputs$"):
        orv.voxel_downsample_with_normals(np.zeros((4, 2)), frame, 1.0)
    with pytest.raises(ValueError, match="^voxel_downsample_with_normals points/normals size mismatch$"):
        orv.voxel_downsample_with_normals(frame, np.zeros((3, 3)), 1.0)
    with pytest.raises(ValueError, match="^voxel_downsample_with_normals voxel_size must be > 0$"):
        orv.voxel_downsample_with_normals(np.zeros((0, 3)), np.zeros((0, 3)), float("nan"))


def test_empty_input_skips_validation():
    for cols in (2, 3, 5):
        out = orv.voxel_downsample_xd(np.zeros((0, cols)), -1.0, 0, 1, 7)
        assert out.shape == (0, cols)
    assert orv.voxel_downsample(np.zeros((0, 3)), -1.0)[0].shape == (0, 3)
    # voxel_downsample validates nothing: with a zero voxel size every coordinate becomes NaN or inf, so
    # every point lands in the INT_MIN voxel
    p, i = orv.voxel_downsample(np.array([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0], [2.0, 2.0, 2.0]]), 0.0)
    assert len(p) == 1
    # a NaN voxel size passes the reference's `voxel_size <= 0` check: one INT_MIN voxel
    assert len(orv.voxel_downsample_xd(np.random.default_rng(0).random((10, 3)), float("nan"), 1, 1, orv.FIRST_N_POINT)) == 1
