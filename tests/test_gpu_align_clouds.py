"""GPU tests of global cloud alignment (ouster-sdk_b200/csrc/ob_align_clouds.cu, DESIGN f-14) against the CPU oracle
(oracle/orc_align_clouds.c) on the scenes of tests/align_scenes.py.

Exact: the feature counts, the grid spec, the target's raw BEV grids and Z histogram, and the confidence counts when
the oracle is given the GPU's poses.  The correlation scores agree within SCORE_TOL (the grids' mean and norm are
summed in a tree on the GPU, in sequence in the oracle); the decisions taken on them (coarse and fine index, Z
shift, dx, dy) are equal wherever the oracle's best beats its runner-up by more than SCORE_TOL, and the scenes are
checked to have that margin.  Poses agree within POSE_TOL per entry (ICP's sums, DESIGN 9)."""
import os
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import align_clouds as oac
from tests import align_scenes as A

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-9
POSE_TOL = 1e-9

CASES = [("room", 37.0, (1.0, -0.5, 0.1)), ("box_island", 137.0, (2.0, 1.0, 0.3)), ("wall", -170.0, (-1.5, 2.0, 0.2)),
         ("open", 0.0, (3.0, -1.0, 0.5))]


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


_pairs = {}


def _pair(name, yaw, t):
    key = (name, yaw, t)
    if key not in _pairs:
        _pairs[key] = A.pair(name, A.pose(yaw, t))
    return _pairs[key]


def _margin(scores):
    s = np.sort(np.asarray(scores))[::-1]
    return s[0] - s[1]


def _compare(g, o, tr_g, tr_o, normals, sp, sn, tp, tn, ob):
    """GPU trace tr_g against oracle trace tr_o for one call."""
    for k in ("source_features", "target_features", "searched", "bound_m", "fine_pixel_m", "coarse_pixel_m",
              "max_shift_m", "fine_base_n", "fine_fft_n", "fine_max_shift", "coarse_base_n", "coarse_fft_n",
              "coarse_max_shift"):
        assert tr_g[k] == tr_o[k], k
    for k in ("target_fine_grid", "target_coarse_grid", "target_z_hist"):
        assert np.array_equal(tr_g[k], tr_o[k]), k
    np.testing.assert_allclose(tr_g["coarse_scores"], tr_o["coarse_scores"], rtol=0, atol=SCORE_TOL)
    np.testing.assert_allclose(tr_g["fine_scores"], tr_o["fine_scores"], rtol=0, atol=SCORE_TOL)
    # the decisions, where the oracle's choice is clear (asserted: the check is not vacuous on these scenes)
    assert _margin(tr_o["coarse_scores"]) > SCORE_TOL
    assert tr_g["coarse_index"] == tr_o["coarse_index"]
    assert _margin(tr_o["fine_scores"]) > SCORE_TOL
    assert tr_g["fine_index"] == tr_o["fine_index"]
    for k in ("fine_z_bins", "fine_dx", "fine_dy"):
        assert np.array_equal(tr_g[k], tr_o[k]), k
    np.testing.assert_allclose(tr_g["initial_pose"], tr_o["initial_pose"], rtol=0, atol=POSE_TOL)
    np.testing.assert_allclose(tr_g["icp_poses"], tr_o["icp_poses"], rtol=0, atol=POSE_TOL)
    np.testing.assert_allclose(g, o, rtol=0, atol=POSE_TOL)
    # the counts, with the oracle at the GPU's poses
    fs, fsn = oac.features(sp, sn if normals else None)
    ft, ftn = oac.features(tp, tn if normals else None)
    for which, pose in (("initial", tr_g["initial_pose"]), ("refined", tr_g["icp_poses"][2])):
        c, m, n = oac.confidence(fs, ft, pose, fsn, ftn)
        assert (tr_g[f"{which}_matched"], tr_g[f"{which}_total"]) == (m, n), which
        assert tr_g[f"{which}_confidence"] == c, which


@pytest.mark.parametrize("name,yaw,t", CASES)
@pytest.mark.parametrize("normals", [False, True])
def test_against_the_oracle(ob, name, yaw, t, normals):
    sp, sn, tp, tn = _pair(name, yaw, t)
    guess = A.pose(yaw + 3.0, (t[0] + 0.4, t[1] - 0.3, t[2])) if name == "box_island" else None
    kw = dict(source_normals=sn, target_normals=tn) if normals else {}
    g, gc, tr_g = ob.core.align_clouds(sp, tp, initial_guess=guess, compute_confidence=True, trace=True, **kw)
    o, oc, tr_o = oac.align_clouds(sp, tp, guess, grids=True, **kw)
    _compare(g, o, tr_g, tr_o, normals, sp, sn, tp, tn, ob)
    assert gc == oc


def test_float32_and_device_inputs(ob):
    import torch
    sp, sn, tp, tn = _pair("room", 37.0, (1.0, -0.5, 0.1))
    s32, t32, sn32, tn32 = (a.astype(np.float32) for a in (sp, tp, sn, tn))
    g, gc, tr_g = ob.core.align_clouds(s32, t32, sn32, tn32, compute_confidence=True, trace=True)
    o, oc, tr_o = oac.align_clouds(s32.astype(np.float64), t32.astype(np.float64), None, sn32.astype(np.float64),
                                   tn32.astype(np.float64), grids=True)
    _compare(g, o, tr_g, tr_o, True, s32.astype(np.float64), sn32.astype(np.float64), t32.astype(np.float64),
             tn32.astype(np.float64), ob)
    for dt in (np.float32, np.float64):
        host = ob.core.align_clouds(sp.astype(dt), tp.astype(dt), sn.astype(dt), tn.astype(dt),
                                    compute_confidence=True)
        dev = [torch.as_tensor(a.astype(dt), device="cuda") for a in (sp, tp, sn, tn)]
        guess = torch.eye(4, dtype=torch.float64, device="cuda")
        pose, conf = ob.core.align_clouds(*dev, initial_guess=guess, compute_confidence=True)
        assert pose.is_cuda and conf.is_cuda
        assert np.array_equal(pose.cpu().numpy(), host[0]) and float(conf.cpu()[0]) == host[1]


def test_device_counts_from_voxel_downsample(ob):
    import torch
    sp, _, tp, _ = _pair("box_island", 137.0, (2.0, 1.0, 0.3))
    bufs, counts, host = [], [], []
    for a in (sp, tp):
        d = torch.as_tensor(a, device="cuda")
        n = torch.tensor([len(a)], dtype=torch.int64, device="cuda")
        pts, _, cnt = ob.core.voxel_downsample(d, 0.05, mode="shuffle_first", n=n)
        bufs.append(pts)
        counts.append(cnt)
        host.append(pts[:int(cnt.cpu()[0])].cpu().numpy())
    pose, conf = ob.core.align_clouds(bufs[0], bufs[1], n_source=counts[0], n_target=counts[1],
                                      compute_confidence=True)
    ref = ob.core.align_clouds(host[0], host[1], compute_confidence=True)
    assert np.array_equal(pose.cpu().numpy(), ref[0]) and float(conf.cpu()[0]) == ref[1]


def _big():
    if "big" not in _pairs:
        _pairs["big"] = A.pair("open", A.pose(137.0, (-2.0, 1.5, 0.2)), 128, 2048)
    return _pairs["big"]


def test_confidence_samples_large_clouds(ob):
    sp, sn, tp, tn = _big()
    g, gc, tr_g = ob.core.align_clouds(sp, tp, sn, tn, compute_confidence=True, trace=True)
    assert tr_g["source_features"] > 16000 and tr_g["target_features"] > 16000
    assert tr_g["refined_total"] == 32000
    o, oc, tr_o = oac.align_clouds(sp, tp, None, sn, tn, grids=True)
    _compare(g, o, tr_g, tr_o, True, sp, sn, tp, tn, ob)
    assert gc == oc


def test_replay_is_bit_identical_and_launches_are_pinned(ob):
    counts = {}
    for normals in (False, True):
        for name, h, w in (("box_island", 32, 512), ("open", 128, 2048)):  # the second samples the confidence
            sp, sn, tp, tn = _big() if name == "open" else _pair("box_island", 137.0, (2.0, 1.0, 0.3))
            kw = dict(source_normals=sn, target_normals=tn) if normals else {}
            before = ob.core.kernel_launch_count("align")
            a = ob.core.align_clouds(sp, tp, compute_confidence=True, trace=True, **kw)
            n = ob.core.kernel_launch_count("align") - before
            b = ob.core.align_clouds(sp, tp, compute_confidence=True, trace=True, **kw)
            assert np.array_equal(a[0], b[0]) and a[1] == b[1]
            for k, v in a[2].items():
                if k == "stage_ms":
                    continue
                assert np.array_equal(np.asarray(v), np.asarray(b[2][k])), k
            counts.setdefault(normals, set()).add(n)
    # the same launches whatever the point count; the figures are this implementation's kernel schedule
    assert counts == {False: {EXPECTED_LAUNCHES[False]}, True: {EXPECTED_LAUNCHES[True]}}, counts


# launches of family "align" per call: features, statistics, target grids and spectra, Z shift, 6 groups of pass 1,
# pass 2, the three ob_cloud_align calls (10 iterations each), the sample masks and the four ob_cloud_nearest calls
# of the confidence
EXPECTED_LAUNCHES = {False: 302, True: 242}


def test_early_return_and_errors(ob):
    rs = np.random.default_rng(2)
    few = rs.normal(size=(15, 3))
    guess = A.pose(20.0, (0.5, 0.25, 0.0))
    pose, conf, tr = ob.core.align_clouds(few, rs.normal(size=(500, 3)) * 5, initial_guess=guess,
                                          compute_confidence=True, trace=True)
    assert np.array_equal(pose, guess) and conf == 0.0 and tr["searched"] == 0 and tr["source_features"] == 15
    nan = np.full((100, 3), np.nan)
    pose, conf = ob.core.align_clouds(nan, nan, initial_guess=guess, compute_confidence=True)
    assert np.array_equal(pose, guess) and conf == 0.0
    with pytest.raises(ValueError, match=r"^source_points must have shape \(N, 3\)$"):
        ob.core.align_clouds(np.zeros((5, 4)), np.zeros((5, 3)))
    with pytest.raises(ValueError, match=r"^target_points and target_normals must have the same number of rows$"):
        ob.core.align_clouds(np.zeros((5, 3)), np.zeros((5, 3)), np.zeros((5, 3)), np.zeros((4, 3)))


def test_pyapi_matches_core_on_both_signatures(ob):
    sp, sn, tp, tn = _pair("room", 37.0, (1.0, -0.5, 0.1))
    guess = A.pose(30.0)
    p = ob.pyapi.align_clouds(sp, tp)
    assert np.array_equal(p, ob.core.align_clouds(sp, tp)[0])
    p, c = ob.pyapi.align_clouds(sp, tp, guess, True)
    assert (p, c) == (p, c) and np.array_equal(p, ob.core.align_clouds(sp, tp, initial_guess=guess)[0])
    assert c == ob.core.align_clouds(sp, tp, initial_guess=guess, compute_confidence=True)[1]
    p, c = ob.pyapi.align_clouds(sp, sn, tp, tn, compute_confidence=True)
    ref = ob.core.align_clouds(sp, tp, sn, tn, compute_confidence=True)
    assert np.array_equal(p, ref[0]) and c == ref[1]
    assert np.array_equal(ob.pyapi.align_clouds(sp, sn, tp, tn, guess), ob.core.align_clouds(sp, tp, sn, tn, guess)[0])


def test_cpp_dropin_example(tmp_path):
    graft.build()
    root = graft.ROOT
    lib_dir = os.path.join(root, "ouster-sdk_b200", "lib")
    exe = str(tmp_path / "align_clouds_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "align_clouds_dropin_example.cpp"), "-L", lib_dir,
                           "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ALIGN CLOUDS DROPIN OK" in out.stdout, (out.stdout, out.stderr)
