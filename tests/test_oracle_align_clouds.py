"""CPU checks of the align_clouds oracle (oracle/orc_align_clouds.c) on scenes whose relative pose is known by
construction (tests/align_scenes.py): truth recovered with and without normals and with and without a guess, every
grid-size branch, the confidence sampling of large clouds, the guard, the early return and the error texts."""
import numpy as np
import pytest

from oracle import align_clouds as oac
from tests import align_scenes as A

MAX_TRANS_M, MAX_ROT_DEG = 0.05, 0.5

# yaw (deg), translation (m, with a Z offset) per scene
WITH_NORMALS = [("room", 37.0, (1.0, -0.5, 0.1)), ("room", -170.0, (0.5, 1.0, 0.0)),
                ("box_island", 137.0, (2.0, 1.0, 0.3)), ("box_island", 0.0, (0.0, 0.0, 0.0)),
                ("wall", -170.0, (-1.5, 2.0, 0.2)), ("wall", 0.0, (3.0, 0.0, 0.3)),
                ("open", 0.0, (3.0, -1.0, 0.5)), ("open", 137.0, (-2.0, 1.5, 0.2))]
# without normals the features are 0.4 m voxel averages, which two scans of a scene sample differently; point-to-point
# ICP then settles a few centimetres off.  These pairs share one scan, moved, so the averages agree.
POINTS_ONLY = [("room", 37.0, (1.0, -0.5, 0.1)), ("room", -170.0, (0.5, 1.0, 0.0)),
               ("box_island", 137.0, (2.0, 1.0, 0.3)), ("wall", -170.0, (-1.5, 2.0, 0.2)),
               ("open", 0.0, (3.0, -1.0, 0.5)), ("open", 137.0, (-2.0, 1.5, 0.2))]

_cache = {}


def _scan(name, h=64, w=1024):
    key = ("scan", name, h, w)
    if key not in _cache:
        _cache[key] = A.scan(name, None, h, w)
    return _cache[key]


def _pair(name, yaw, t):
    key = ("pair", name, yaw, t)
    if key not in _cache:
        _cache[key] = A.pair(name, A.pose(yaw, t), 64, 1024)
    return _cache[key]


def _moved(name, truth):
    """The target scan and the same points moved by inv(truth), with 2 mm of noise."""
    tp, _ = _scan(name)
    ti = np.linalg.inv(truth)
    sp = tp @ ti[:3, :3].T + ti[:3, 3] + np.random.default_rng(3).normal(0.0, 0.002, tp.shape)
    return sp, tp


def _check(pose, truth):
    e_t, e_r = A.pose_error(pose, truth)
    assert e_t <= MAX_TRANS_M and e_r <= MAX_ROT_DEG, (e_t, e_r)


@pytest.mark.parametrize("name,yaw,t", WITH_NORMALS)
@pytest.mark.parametrize("with_guess", [False, True])
def test_recovers_the_truth_with_normals(name, yaw, t, with_guess):
    truth = A.pose(yaw, t)
    sp, sn, tp, tn = _pair(name, yaw, t)
    pose, conf, tr = oac.align_clouds(sp, tp, truth if with_guess else None, sn, tn)
    _check(pose, truth)
    assert 0.3 < conf <= 1.0 and tr["searched"] == 1


@pytest.mark.parametrize("name,yaw,t", POINTS_ONLY)
@pytest.mark.parametrize("with_guess", [False, True])
def test_recovers_the_truth_from_points_only(name, yaw, t, with_guess):
    truth = A.pose(yaw, t)
    sp, tp = _moved(name, truth)
    pose, conf, _ = oac.align_clouds(sp, tp, truth if with_guess else None)
    _check(pose, truth)
    assert 0.5 < conf <= 1.0


def test_grid_branches():
    """bound <= 18 m: 0.20 m pixels; <= 30 m: 0.15 m; larger: 0.25 m.  The coarse grid is 0.5 m throughout."""
    seen = {}
    for name in ("room", "box_island", "wall", "open"):
        sp, _, tp, _ = _pair(name, *{"room": (37.0, (1.0, -0.5, 0.1)), "box_island": (137.0, (2.0, 1.0, 0.3)),
                                     "wall": (-170.0, (-1.5, 2.0, 0.2)), "open": (0.0, (3.0, -1.0, 0.5))}[name])
        _, _, tr = oac.align_clouds(sp, tp)
        b = tr["bound_m"]
        assert 10.0 <= b <= 60.0 and tr["coarse_pixel_m"] == 0.5
        px = 0.20 if b <= 18.0 else (0.15 if b <= 30.0 else 0.25)
        assert tr["fine_pixel_m"] == px
        for g in ("fine", "coarse"):
            base = max(8, int(np.ceil(2.0 * b / tr[f"{g}_pixel_m"])) + 1)
            assert tr[f"{g}_base_n"] == base
            fft = 1 << int(np.ceil(np.log2(2 * base - 1)))
            shift = max(1, int(np.floor(max(0.1, tr["max_shift_m"]) / tr[f"{g}_pixel_m"] + 0.5)))
            assert tr[f"{g}_fft_n"] == max(8, fft) and tr[f"{g}_max_shift"] == min(shift, base // 2)
        seen[px] = b
    assert set(seen) == {0.20, 0.15, 0.25}, seen
    assert max(seen.values()) > 30.0


def test_a_far_guess_widens_the_grid():
    sp, _, tp, _ = _pair("room", 37.0, (1.0, -0.5, 0.1))
    guess = A.pose(0.0, (45.0, 0.0, 0.0))
    _, _, tr = oac.align_clouds(sp, tp, guess)
    assert tr["bound_m"] == 47.0 and tr["fine_pixel_m"] == 0.25
    _, _, tr = oac.align_clouds(sp, tp, A.pose(0.0, (70.0, 0.0, 0.0)))
    assert tr["bound_m"] == 60.0 and tr["fine_base_n"] == 481 and tr["coarse_base_n"] == 241


def test_large_clouds_sample_the_confidence():
    sp, sn, tp, tn = A.pair("open", A.pose(137.0, (-2.0, 1.5, 0.2)), 128, 2048)
    pose, conf, tr = oac.align_clouds(sp, tp, None, sn, tn)
    assert tr["source_features"] > 16000 and tr["target_features"] > 16000
    assert tr["initial_total"] == tr["refined_total"] == 32000
    _check(pose, A.pose(137.0, (-2.0, 1.5, 0.2)))


def test_confidence_counts_and_guard():
    sp, sn, tp, tn = _pair("box_island", 137.0, (2.0, 1.0, 0.3))
    pose, conf, tr = oac.align_clouds(sp, tp, None, sn, tn)
    fs, fsn = oac.features(sp, sn)
    ft, ftn = oac.features(tp, tn)
    c, m, n = oac.confidence(fs, ft, tr["icp_poses"][2], fsn, ftn)
    assert (c, m, n) == (tr["refined_confidence"], tr["refined_matched"], tr["refined_total"])
    assert n == len(fs) + len(ft) and conf == c
    # compute_confidence=False: the same pose, confidence 0
    p2, c2, _ = oac.align_clouds(sp, tp, None, sn, tn, compute_confidence=False)
    assert np.array_equal(p2, pose) and c2 == 0.0
    # the guard: a wrong pose scores lower than the search's, so the refined pose must not be worse
    far = A.pose(90.0, (5.0, 0.0, 0.0)) @ tr["icp_poses"][2]
    c_far = oac.confidence(fs, ft, far, fsn, ftn)[0]
    assert c_far + 1e-6 < tr["refined_confidence"]
    assert tr["refined_confidence"] + 1e-6 >= tr["initial_confidence"] or np.array_equal(pose, tr["initial_pose"])


def test_guard_returns_the_search_pose_when_icp_loses_overlap():
    """A scene where ICP drifts: the oracle must return the search pose whenever refined + 1e-6 < initial."""
    hits = 0
    for name, yaw, t in POINTS_ONLY + WITH_NORMALS:
        sp, sn, tp, tn = _pair(name, yaw, t)
        pose, conf, tr = oac.align_clouds(sp, tp)
        if tr["refined_confidence"] + 1e-6 < tr["initial_confidence"]:
            hits += 1
            assert np.array_equal(pose, tr["initial_pose"]) and conf == tr["initial_confidence"]
        else:
            assert np.array_equal(pose, tr["icp_poses"][2]) and conf == tr["refined_confidence"]
    assert hits > 0


def test_fewer_than_20_features_return_the_guess_bit_for_bit():
    rs = np.random.default_rng(5)
    guess = A.pose(33.0, (0.3, -0.2, 0.1))
    guess[0, 1] += 1e-17  # any bits at all come back
    few = rs.normal(size=(19, 3)) * 10.0
    many = rs.normal(size=(2000, 3)) * 10.0
    for s, t in ((few, many), (many, few), (few, few)):
        pose, conf, tr = oac.align_clouds(s, t, guess)
        assert np.array_equal(pose, guess) and conf == 0.0 and tr["searched"] == 0
    # 25 points in one 0.4 m voxel are one feature
    dense = rs.uniform(0.01, 0.39, size=(25, 3))
    pose, conf, tr = oac.align_clouds(dense, many, guess)
    assert tr["source_features"] == 1 and np.array_equal(pose, guess) and conf == 0.0


def test_all_nan_and_invalid_normals():
    nan = np.full((200, 3), np.nan)
    guess = A.pose(10.0, (1.0, 0.0, 0.0))
    pose, conf, tr = oac.align_clouds(nan, nan, guess)
    assert np.array_equal(pose, guess) and conf == 0.0 and tr["source_features"] == 0
    sp, sn, tp, tn = _pair("room", 37.0, (1.0, -0.5, 0.1))
    bad = sn.copy()
    bad[:] = 0.0  # norm <= 1e-12: every source row is dropped
    pose, conf, tr = oac.align_clouds(sp, tp, guess, bad, tn)
    assert tr["source_features"] == 0 and np.array_equal(pose, guess)


def test_error_texts_in_the_reference_order():
    ok, n3 = np.zeros((5, 3)), np.zeros((5, 3))
    with pytest.raises(ValueError, match=r"^source_points must have shape \(N, 3\)$"):
        oac.align_clouds(np.zeros((5, 2)), np.zeros((5, 4)))
    with pytest.raises(ValueError, match=r"^source_normals must have shape \(N, 3\)$"):
        oac.align_clouds(ok, np.zeros((5, 4)), None, np.zeros((5, 2)), n3)
    with pytest.raises(ValueError, match=r"^source_points and source_normals must have the same number of rows$"):
        oac.align_clouds(ok, np.zeros((5, 4)), None, np.zeros((4, 3)), n3)
    with pytest.raises(ValueError, match=r"^target_points must have shape \(N, 3\)$"):
        oac.align_clouds(ok, np.zeros((5, 4)), None, n3, n3)
    with pytest.raises(ValueError, match=r"^target_points and target_normals must have the same number of rows$"):
        oac.align_clouds(ok, ok, None, n3, np.zeros((6, 3)))
