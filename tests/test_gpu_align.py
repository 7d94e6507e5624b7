"""GPU tests of cloud-to-cloud ICP (ouster-sdk_b200/csrc/ob_align.cu) against the CPU oracle (oracle/orc_align.c):
the nearest-neighbour search bit for bit, point_to_point_align / point_to_plane_align with the oracle's iteration
count and every pose entry within POSE_TOL (the device sums run in a tree, the oracle's in sequence; DESIGN 9)."""
import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import align as oa
from tests.test_oracle_normals import room_scene

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-12


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def rot(axis_angle):
    from scipy.spatial.transform import Rotation
    return Rotation.from_rotvec(axis_angle).as_matrix()


def wall_normals(d):
    """inward unit normal of the cube wall each beam of room_scene hits"""
    axis = np.argmax(np.abs(d), axis=-1)
    e = np.zeros_like(d)
    np.put_along_axis(e, axis[..., None], -np.sign(np.take_along_axis(d, axis[..., None], -1)), -1)
    return e


def room_pair(h=64, w=512, seed=0, noise=0.002):
    """(source, target, source normals, target normals, truth): a 10 m room seen from two poses; the source is the
    target moved by inv(truth) plus noise.  The floor and ceiling are out of view, so z is not observable."""
    rs = np.random.default_rng(seed)
    xyz, _, d = room_scene(h, w, half=10000.0)
    tgt = xyz.reshape(-1, 3)
    nt = wall_normals(d).reshape(-1, 3)
    truth = np.eye(4)
    truth[:3, :3] = rot(np.radians([0.3, -0.2, 1.0]))
    truth[:3, 3] = [0.12, -0.07, 0.0]
    ti = np.linalg.inv(truth)
    src = tgt @ ti[:3, :3].T + ti[:3, 3] + rs.normal(0, noise, tgt.shape)
    ns = nt @ ti[:3, :3].T + rs.normal(0, 0.01, nt.shape)
    return src, tgt, ns, nt, truth


def quantised_cloud(rs, n, step=0.05, extent=2.0):
    return np.round(rs.uniform(-extent, extent, (n, 3)) / step) * step


def poison(rs, a):
    a = a.copy()
    for v in (np.nan, np.inf, -np.inf, 1e300, -1e300):
        rows = rs.choice(len(a), 50, replace=False)
        a[rows, rs.integers(0, 3, 50)] = v
    return a


@pytest.mark.parametrize("mcd", [0.05, 0.3, 2.0])
@pytest.mark.parametrize("with_normals", [False, True])
def test_cloud_nearest_bit_exact_on_a_quantised_grid(ob, mcd, with_normals):
    rs = np.random.default_rng(int(mcd * 100) + with_normals)
    tgt = poison(rs, quantised_cloud(rs, 100_000))
    qry = poison(rs, quantised_cloud(rs, 100_000) + rs.choice([0.0, 0.025], (100_000, 3)))
    nrm = None
    if with_normals:
        nrm = rs.normal(size=tgt.shape)
        bad = rs.choice(len(nrm), 5000, replace=False)
        nrm[bad[:2000]] = 0.0
        nrm[bad[2000:3000]] = 1e-13
        nrm[bad[3000:4000], 0] = np.nan
        nrm[bad[4000:], 1] = np.inf
    want = oa.cloud_nearest(tgt, qry, mcd, mcd * mcd, nrm)
    got = ob.cloud_nearest(tgt, qry, mcd, mcd * mcd, target_normals=nrm)
    assert np.array_equal(got, want)
    assert (want >= 0).mean() > 0.3 and (want < 0).any()
    import torch
    dev = torch.device("cuda", 0)
    gd = ob.cloud_nearest(torch.from_numpy(tgt).to(dev), torch.from_numpy(qry).to(dev), mcd, mcd * mcd,
                          target_normals=None if nrm is None else torch.from_numpy(nrm).to(dev))
    assert np.array_equal(gd.cpu().numpy(), want)


def test_cloud_nearest_float32_and_ties(ob):
    # equal distances: (0.5, 0.5, 0.5) is 0.5 from both rows; the cell visited first (dx = -1) wins, and inside one
    # cell the lower row wins
    tgt = np.array([[0.5, 0.5, 0.0], [0.5, 0.5, 1.0], [0.5, 0.5, 1.0], [-0.5, 0.5, 0.5]], np.float64)
    tgt = np.vstack([tgt, np.full((30, 3), 50.0)])
    qry = np.array([[0.5, 0.5, 0.5], [0.5, 0.5, 0.9], [0.0, 0.5, 0.5]])
    want = oa.cloud_nearest(tgt, qry, 1.0, 1.0)
    assert np.array_equal(ob.cloud_nearest(tgt, qry, 1.0, 1.0), want)
    assert list(want) == [0, 1, 3]
    rs = np.random.default_rng(5)
    t32, q32 = quantised_cloud(rs, 20_000).astype(np.float32), quantised_cloud(rs, 20_000).astype(np.float32)
    assert np.array_equal(ob.cloud_nearest(t32, q32, 0.1, 0.01), oa.cloud_nearest(t32, q32, 0.1, 0.01))


def _both(ob, mode, src, tgt, ns, nt, guess, **kw):
    if mode == "p2p":
        want, wit = oa.point_to_point_align(src, tgt, guess, **kw)
        got, git = ob.cloud_align(src, tgt, initial_guess=guess, **kw)
    else:
        want, wit = oa.point_to_plane_align(src, tgt, ns, nt, guess, **kw)
        got, git = ob.cloud_align(src, tgt, ns, nt, initial_guess=guess, **kw)
    return want, wit, got, git


@pytest.mark.parametrize("mode", ["p2p", "plane"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("with_guess", [False, True])
def test_align_room_scene_vs_oracle_and_truth(ob, mode, dtype, with_guess):
    src, tgt, ns, nt, truth = room_pair()
    src, tgt, ns, nt = (a.astype(dtype) for a in (src, tgt, ns, nt))
    guess = None
    if with_guess:
        guess = np.eye(4)
        guess[:3, :3] = rot(np.radians([0.0, 0.0, 0.7]))
        guess[:3, 3] = [0.1, -0.05, 0.0]
    want, wit, got, git = _both(ob, mode, src, tgt, ns, nt, guess, max_corr_dist=0.5)
    print(f"{mode} {np.dtype(dtype).name} guess={with_guess}: iterations {git}, max |gpu - oracle| "
          f"{np.abs(got - want).max():.3e}")
    assert git == wit and git >= 2
    assert np.abs(got - want).max() <= POSE_TOL
    err = got @ np.linalg.inv(truth)
    from scipy.spatial.transform import Rotation
    assert np.linalg.norm(Rotation.from_matrix(err[:3, :3]).as_rotvec()) < 2e-4
    assert np.linalg.norm(err[:2, 3]) < 2e-3


def test_reference_known_answers_through_pyapi(ob):
    api = ob.pyapi
    src = np.array([[x, y, z] for x in (-1.0, 0.0, 1.0) for y in (-1.0, 0.0, 1.0) for z in (-1.0, 0.0, 1.0)])
    t = np.array([0.1, -0.05, 0.025])
    got = api.point_to_point_align(src, np.ascontiguousarray(src + t), max_corr_dist=0.5)
    assert isinstance(got, np.ndarray) and got.shape == (4, 4) and got.dtype == np.float64
    np.testing.assert_allclose(got[:3, :3], np.eye(3), atol=1e-10)
    np.testing.assert_allclose(got[:3, 3], t, atol=1e-10)
    # the plane case is exactly degenerate: rotation about z and x, y translation are unconstrained, and the 1e-10
    # diagonal with the LDLT's pivoting decides the answer
    s = np.array([[x, y, 0.0] for x in range(5) for y in range(5)], np.float64)
    tg = s.copy()
    tg[:, 2] = 0.2
    n = np.tile([0.0, 0.0, 1.0], (25, 1))
    got = api.point_to_plane_align(s, tg, n, n, max_corr_dist=0.5)
    np.testing.assert_allclose(got[:3, :3], np.eye(3), atol=1e-10)
    np.testing.assert_allclose(got[:3, 3], [0.0, 0.0, 0.2], atol=1e-9)
    want, _ = oa.point_to_plane_align(s, tg, n, n, max_corr_dist=0.5)
    assert np.abs(got - want).max() <= POSE_TOL


def test_edge_cases_return_the_guess_bit_for_bit(ob):
    rs = np.random.default_rng(2)
    guess = np.eye(4)
    guess[:3, :3] = rot([0.1, -0.2, 0.3])
    guess[:3, 3] = [1.0 / 3.0, -2.0 / 7.0, np.pi]
    pts = rs.normal(size=(19, 3))
    nrm = rs.normal(size=(19, 3))
    big = rs.normal(size=(200, 3))
    # fewer than 20 rows in either cloud
    for s, t in ((pts, big), (big, pts)):
        got, it = ob.cloud_align(s, t, initial_guess=guess)
        assert np.array_equal(got, guess) and it == 0
    got, it = ob.cloud_align(pts, big, nrm, rs.normal(size=(200, 3)), initial_guess=guess)
    assert np.array_equal(got, guess) and it == 0
    # no correspondence at the first iteration
    got, it = ob.cloud_align(big, big + 100.0, initial_guess=guess)
    assert np.array_equal(got, guess) and it == 0
    # every normal invalid
    zero = np.zeros_like(big)
    got, it = ob.cloud_align(big, big, zero, rs.normal(size=big.shape), initial_guess=guess)
    assert np.array_equal(got, guess) and it == 0
    got, it = ob.cloud_align(big, big, rs.normal(size=big.shape), np.full_like(big, np.nan), initial_guess=guess)
    assert np.array_equal(got, guess) and it == 0


@pytest.mark.parametrize("angle", [0.0, 180.0])
def test_normal_gate_limits_match_the_oracle(ob, angle):
    src, tgt, ns, nt, _ = room_pair(32, 256, seed=4)
    want, wit, got, git = _both(ob, "plane", src, tgt, ns, nt, None, max_corr_dist=0.5, max_normal_angle_deg=angle)
    assert git == wit
    assert np.abs(got - want).max() <= POSE_TOL


def test_errors_in_the_reference_order(ob):
    api = ob.pyapi
    s = np.zeros((25, 3))
    with pytest.raises(ValueError, match="max_corr_dist must be finite and greater than zero"):
        api.point_to_point_align(s, s, max_corr_dist=0.0)
    with pytest.raises(ValueError, match="max_corr_dist must be finite and greater than zero"):
        api.point_to_plane_align(s, s, s[:3], s, max_corr_dist=np.inf, max_normal_angle_deg=-1.0)
    with pytest.raises(ValueError, match=r"max_normal_angle_deg must be finite and in \[0, 180\]"):
        api.point_to_plane_align(s, s, s[:3], s, max_normal_angle_deg=np.nan)
    with pytest.raises(ValueError, match="source_points and source_normals must have the same number of rows"):
        api.point_to_plane_align(s, s, s[:3], s[:4])
    with pytest.raises(ValueError, match="target_points and target_normals must have the same number of rows"):
        api.point_to_plane_align(s, s, s, s[:4])


def test_device_chain_matches_the_host_path_and_replays_in_a_graph(ob):
    """XYZ -> ob_normals -> voxel_downsample_with_normals (device count) -> point_to_plane_align with device counts
    and a device pose, against the same steps with host counts; then the align replayed from a CUDA graph."""
    import torch
    dev = torch.device("cuda", 0)
    h, w = 64, 1024
    xyz_t, rng_t, d = room_scene(h, w, half=10000.0)
    truth = np.eye(4)
    truth[:3, :3] = rot(np.radians([0.0, 0.0, 0.8]))
    truth[:3, 3] = [0.05, 0.02, 0.0]
    st = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
    clouds_dev, clouds_host = [], []
    for k, pose in enumerate((np.eye(4), np.linalg.inv(truth))):
        xyz = (xyz_t.reshape(-1, 3) @ pose[:3, :3].T + pose[:3, 3]).reshape(h, w, 3)
        origins = np.repeat(pose[None, :3, 3], w, 0)
        x = torch.from_numpy(xyz).to(dev)
        r = torch.from_numpy(rng_t.view(np.int32)).to(dev)
        nd = ob.normals(x, r, sensor_origins_xyz=origins, stream=st)
        cnt = torch.full((1,), h * w, dtype=torch.int64, device=dev)
        p, n, _, c = ob.voxel_downsample(x.reshape(-1, 3), 0.3, "point_normal", normals=nd.reshape(-1, 3), n=cnt,
                                         stream=st)
        clouds_dev.append((p, n, c))
        nh = ob.normals(xyz, rng_t, sensor_origins_xyz=origins)
        ph, nh2, _ = ob.voxel_downsample(xyz.reshape(-1, 3), 0.3, "point_normal", normals=nh.reshape(-1, 3))
        clouds_host.append((ph, nh2))
    (tp, tn, tc), (sp, sn, sc) = clouds_dev
    guess = torch.eye(4, dtype=torch.float64, device=dev)
    pose_d, it_d = ob.cloud_align(sp, tp, sn, tn, initial_guess=guess, max_corr_dist=0.6, n_source=sc, n_target=tc,
                                  stream=st)
    (th, thn), (sh, shn) = clouds_host
    pose_h, it_h = ob.cloud_align(sh, th, shn, thn, max_corr_dist=0.6)
    assert np.array_equal(pose_d.cpu().numpy(), pose_h) and int(it_d.item()) == it_h
    want, wit = oa.point_to_plane_align(sh, th, shn, thn, None, 0.6)
    assert it_h == wit and np.abs(pose_h - want).max() <= POSE_TOL
    # the same call twice, then from a CUDA graph
    again, _ = ob.cloud_align(sp, tp, sn, tn, initial_guess=guess, max_corr_dist=0.6, n_source=sc, n_target=tc,
                              stream=st)
    assert torch.equal(again, pose_d)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    cs = torch.cuda.Stream()
    st_cs = ob.Stream(0, cuda_stream=cs.cuda_stream)
    with torch.cuda.stream(cs):
        ob.cloud_align(sp, tp, sn, tn, initial_guess=guess, max_corr_dist=0.6, n_source=sc, n_target=tc, stream=st_cs)
        cs.synchronize()
        try:
            with torch.cuda.graph(g, stream=cs, capture_error_mode="thread_local"):
                gp, git = ob.cloud_align(sp, tp, sn, tn, initial_guess=guess, max_corr_dist=0.6, n_source=sc,
                                         n_target=tc, stream=st_cs)
        except Exception:
            print("capture failed:", ob._capi.lib.ob_last_error().decode())
            raise
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gp, pose_d) and torch.equal(git, it_d)
    assert ob.kernel_launch_count("align") > 0
