"""GPU tests of frame-to-map registration (ouster-sdk_b200/csrc/ob_voxel_map.cu) against the CPU oracle
(oracle/orc_icp.c): the map and the closest-neighbour search bit for bit including order, build_linear_system bit
for bit, align_points_to_map to 1e-12 (device sin/cos differ from libm in the last bit, DESIGN 9)."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import icp as oi
from oracle import voxel as orv
from tests.test_oracle_normals import room_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def scene(h=128, w=2048, seed=0):
    rs = np.random.default_rng(seed)
    _, rng, d = room_scene(h, w)
    rng = (rng.astype(np.int64) + rs.integers(-40, 41, rng.shape)).astype(np.float64)
    return (d * rng[..., None] * 0.001).reshape(-1, 3)


def rot(axis_angle):
    from scipy.spatial.transform import Rotation
    return Rotation.from_rotvec(axis_angle).as_matrix()


def same_map(gm, om):
    assert gm.size() == om.size()
    assert np.array_equal(gm.point_cloud(), om.point_cloud(), equal_nan=True)


@pytest.mark.parametrize("max_pts", [1, 3, 20])
def test_map_add_remove_extract_bit_exact_over_many_cycles(ob, max_pts):
    rs = np.random.default_rng(max_pts)
    vs, md = 0.5, 6.0
    gm, om = ob.VoxelMap(vs, md, max_pts), oi.VoxelHashMap3d(vs, md, max_pts)
    for cycle in range(110):
        centre = np.array([np.cos(cycle / 9.0), np.sin(cycle / 7.0), 0.1 * cycle]) * 8.0
        n = int(rs.integers(0, 3000))
        pts = centre + rs.normal(0, 3.0, (n, 3))
        if cycle % 10 == 3:                       # one dense voxel
            pts[: n // 2] = centre + rs.random((n // 2, 3)) * 0.49
        dtype = np.float32 if cycle % 2 else np.float64
        if cycle % 17 == 5 and n > 4:             # rows in the INT32_MIN voxel
            big = 1e300 if dtype == np.float64 else 3e38
            pts[0, 0], pts[1, 1], pts[2] = np.nan, big, [-big, np.nan, big]
        pts = pts.astype(dtype)
        gm.add_points(pts)
        om.add_points(pts.astype(np.float64))
        if cycle % 3 == 0:
            got = gm.remove_far(centre, extract=True)
            want = om.extract_voxels_far_from_location(centre)
            assert np.array_equal(got, want, equal_nan=True), cycle
        elif cycle % 3 == 1:
            gm.remove_far(centre)
            om.remove_voxels_far_from_location(centre)
        same_map(gm, om)
    gm.clear()
    om.clear()
    same_map(gm, om)


def test_closest_neighbors_bit_exact_with_and_without_bound(ob):
    pts = scene(64, 1024)
    gm, om = ob.VoxelMap(0.5, 100.0, 20), oi.VoxelHashMap3d(0.5, 100.0, 20)
    gm.add_points(pts)
    om.add_points(pts)
    rs = np.random.default_rng(5)
    q = pts[rs.integers(0, len(pts), 3000)] + rs.normal(0, 0.4, (3000, 3))
    for bound in (oi.DBL_MAX, 0.25, 1e-4):
        nb, d2 = gm.closest_neighbors(q, bound)
        wnb, wd2 = om.get_closest_neighbors(q, bound)
        assert np.array_equal(nb, wnb) and np.array_equal(d2, wd2), bound
    # float32 queries are widened exactly
    nb, d2 = gm.closest_neighbors(q.astype(np.float32))
    wnb, wd2 = om.get_closest_neighbors(q.astype(np.float32).astype(np.float64))
    assert np.array_equal(nb, wnb) and np.array_equal(d2, wd2)


def test_closest_ties_in_different_voxels_first_shift_wins(ob):
    # the query sits on a voxel face: equal distances in voxel (0,0,0) shift order +x before -x
    m_pts = np.array([[1.25, 0.5, 0.5], [0.75, 0.5, 0.5], [-0.25, 0.5, 0.5]])
    gm, om = ob.VoxelMap(1.0, 100.0, 20), oi.VoxelHashMap3d(1.0, 100.0, 20)
    gm.add_points(m_pts)
    om.add_points(m_pts)
    q = np.array([[1.0, 0.5, 0.5], [0.5, 0.5, 0.5], [0.25, 0.5, 0.5], [9.0, 9.0, 9.0]])
    nb, d2 = gm.closest_neighbors(q)
    wnb, wd2 = om.get_closest_neighbors(q)
    assert np.array_equal(nb, wnb) and np.array_equal(d2, wd2)
    assert np.array_equal(nb[0], [1.25, 0.5, 0.5]) and d2[0] == 0.0625     # own voxel visited first
    assert np.array_equal(nb[3], [0, 0, 0]) and d2[3] == oi.DBL_MAX
    # query in an empty voxel, equal distances in +x and -x: shift (1,0,0) precedes (-1,0,0)
    tm = ob.VoxelMap(1.0, 100.0, 20)
    tm.add_points(np.array([[-0.25, 0.5, 0.5], [1.25, 0.5, 0.5]]))
    nb, d2 = tm.closest_neighbors(np.array([[0.5, 0.5, 0.5]]))
    assert np.array_equal(nb[0], [1.25, 0.5, 0.5]) and d2[0] == 0.5625
    e = ob.VoxelMap(1.0)
    nb, d2 = e.closest_neighbors(q, 2.0)
    assert np.array_equal(nb, np.zeros((4, 3))) and np.array_equal(d2, np.full(4, 2.0))


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000, 100000])
def test_build_linear_system_bit_exact(ob, n):
    rs = np.random.default_rng(n)
    src = rs.random((n, 3)) * 40 - 20
    tgt = src + rs.normal(0, 0.2, (n, 3))
    jtj, jtr = ob.icp_linear_system(src, tgt, 0.37)
    wj, wr = oi.build_linear_system(src, tgt, 0.37)
    assert np.array_equal(jtj, wj) and np.array_equal(jtr, wr)


def _align_both(ob, map_pts, frame, md, ks, iters, vs=1.0, max_pts=20, crit=1e-4):
    gm, om = ob.VoxelMap(vs, 100.0, max_pts), oi.VoxelHashMap3d(vs, 100.0, max_pts)
    if len(map_pts):
        gm.add_points(map_pts)
        om.add_points(map_pts)
    pose, it = ob.icp_align(gm, frame, md, ks, iters, crit)
    wpose, wit = oi.align_points_to_map(frame, om, md, ks, iters, crit)
    return pose, it, wpose, wit


def test_align_known_answers(ob):
    pts = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    shifted = pts + np.array([0.05, 0.02, -0.01])
    pose, it, wpose, wit = _align_both(ob, pts, shifted, 0.5, 0.1, 20, vs=0.5)
    assert it == wit and np.abs(pose - wpose).max() <= 1e-12
    rec = (pose[:3, :3] @ shifted.T).T + pose[:3, 3]
    np.testing.assert_allclose(rec, pts, atol=0.05)
    # empty map: identity, no iteration; no correspondences: one identity step
    pose, it, _, _ = _align_both(ob, np.empty((0, 3)), shifted, 1.0, 0.1, 5, vs=0.5)
    assert it == 0 and np.array_equal(pose, np.eye(4))
    pose, it, wpose, wit = _align_both(ob, pts, shifted + 50.0, 0.5, 0.1, 5, vs=0.5)
    assert it == wit == 1 and np.array_equal(pose, np.eye(4)) and np.array_equal(wpose, np.eye(4))


@pytest.mark.parametrize("iters", [1, 50, 500])
def test_align_room_scene_vs_oracle_and_truth(ob, iters):
    cloud = scene()
    f1, _ = orv.voxel_downsample(cloud, 0.5)
    src, _ = orv.voxel_downsample(f1, 1.5)
    map_pts = f1
    truth = np.eye(4)
    truth[:3, :3] = rot(np.radians([0.4, -0.7, 1.2]))
    truth[:3, 3] = [0.03, -0.02, 0.015]
    moved = (np.linalg.inv(truth)[:3, :3] @ src.T).T + np.linalg.inv(truth)[:3, 3]
    pose, it, wpose, wit = _align_both(ob, map_pts, moved, 1.0, 0.3, iters, vs=0.5, crit=1e-4 if iters != 500 else 1e-12)
    diff = np.abs(pose - wpose).max()
    print(f"iterations {it} (oracle {wit}), max |pose - oracle| = {diff:.3e}")
    assert it == wit and diff <= 1e-12
    if iters > 1:
        err_gpu = np.abs(pose - truth).max()
        err_orc = np.abs(wpose - truth).max()
        assert err_gpu <= err_orc + 1e-9 and err_orc < 0.02, (err_gpu, err_orc)


def test_device_chain_matches_the_host_path_and_replays_in_a_graph(ob):
    """ob_dewarp_frames (device count) -> 2x voxel_downsample (device counts) -> align (device pose) -> transform +
    add_points -> cull, over 5 frames of the room scene, against the same steps with host counts; then align on the
    built map inside a CUDA graph."""
    import torch
    capi = ob._capi
    dev = torch.device("cuda", 0)
    h, w = 64, 1024
    _, rng, d = room_scene(h, w)
    lut = ob.XYZLutT.from_arrays(np.ascontiguousarray(d.reshape(-1, 3)), np.zeros((h * w, 3)), h, w)
    status = np.ones(w, np.uint32)
    step = np.eye(4)
    step[:3, :3] = rot(np.radians([0.0, 0.0, 0.8]))
    step[:3, 3] = [0.04, 0.01, 0.0]
    vs, md = 0.5, 30.0
    gm, hm = ob.VoxelMap(vs, md, 20), ob.VoxelMap(vs, md, 20)
    poses_dev, poses_host = [], []
    st = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
    noise = np.random.default_rng(3)
    for k in range(1, 6):
        r = (rng.astype(np.int64) + noise.integers(-30, 31, rng.shape)).astype(np.uint32)
        poses = np.repeat(np.linalg.matrix_power(step, k)[None], w, 0)      # body_to_world of every column
        keep = [torch.from_numpy(a).to(dev) for a in (r.view(np.int32), poses, status.view(np.int32))]
        frames = (capi.DewarpFramesIO * 1)()
        frames[0].lut, frames[0].range, frames[0].poses, frames[0].status = lut._h, *(x.data_ptr() for x in keep)
        pts = torch.empty((h * w, 3), dtype=torch.float64, device=dev)
        n = torch.zeros(1, dtype=torch.int64, device=dev)
        capi.check(capi.lib.ob_dewarp_frames(frames, 1, 0.5, 100.0, pts.data_ptr(), h * w, None, None, None, None,
                                             C.cast(n.data_ptr(), C.POINTER(C.c_size_t)), st.h))
        p1, _, c1 = ob.voxel_downsample(pts, 0.5 * vs, n=n, stream=st)
        p2, _, c2 = ob.voxel_downsample(p1, 1.5 * vs, n=c1, stream=st)
        pose, it = ob.icp_align(gm, p2, 3.0, 1.0, 50, n=c2, stream=st)
        gm.add_points(ob.transform(p1, pose, stream=st), n=c1, stream=st)
        gm.remove_far(pose[:3, 3].contiguous(), stream=st)
        poses_dev.append(pose.cpu().numpy())
        # host path
        cloud = ob.dewarp_frames([{"lut": lut, "range": r, "poses": poses, "status": status}], 0.5, 100.0)
        assert int(n.item()) == len(cloud)
        h1, _ = ob.voxel_downsample(cloud, 0.5 * vs)
        h2, _ = ob.voxel_downsample(h1, 1.5 * vs)
        hp, _ = ob.icp_align(hm, h2, 3.0, 1.0, 50)
        hm.add_points(ob.transform(h1, hp))
        hm.remove_far(hp[:3, 3])
        poses_host.append(hp)
    for a, b in zip(poses_dev, poses_host):
        assert np.array_equal(a, b)
    assert gm.size() == hm.size()
    assert np.array_equal(gm.point_cloud(), hm.point_cloud())
    # align on the built map, captured into a CUDA graph and replayed
    src = torch.from_numpy(h2).to(dev)
    ref_pose, ref_it = ob.icp_align(gm, src, 3.0, 1.0, 50)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    cs = torch.cuda.Stream()
    st_cs = ob.Stream(0, cuda_stream=cs.cuda_stream)   # wrapped before the capture starts
    with torch.cuda.stream(cs):
        ob.icp_align(gm, src, 3.0, 1.0, 50, stream=st_cs)
        cs.synchronize()
        try:
            with torch.cuda.graph(g, stream=cs, capture_error_mode="thread_local"):
                gp, git = ob.icp_align(gm, src, 3.0, 1.0, 50, stream=st_cs)
        except Exception:
            print("capture failed:", ob._capi.lib.ob_last_error().decode())
            raise
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gp, ref_pose) and torch.equal(git, ref_it)
    assert ob.kernel_launch_count("icp") > 0 and ob.kernel_launch_count("voxel_map") > 0


def test_python_api_names_defaults_and_errors(ob):
    api = ob.pyapi
    m = api.VoxelHashMap3d()
    assert m.empty and m.max_points_per_voxel() == 20 and m.min_pts_threshold() == 1
    with pytest.raises(ValueError, match="add_points expects an Nx3 array"):
        m.add_points(np.zeros((4, 2)))
    with pytest.raises(ValueError, match="VoxelHashMap method expects a 3-element point"):
        m.get_closest_neighbor(np.zeros(2))
    pts = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    m = api.VoxelHashMap3d(voxel_size=0.5, max_distance=10.0)
    m.add_points(pts)
    assert not m.empty
    nb, d2 = m.get_closest_neighbor(np.array([0.9, 0.0, 0.0]))
    assert np.array_equal(nb, [1, 0, 0]) and d2 == pytest.approx(0.01)
    reg = api.ICPRegistration(max_num_iterations=20)
    t = reg.align_points_to_map(pts + [0.05, 0.02, -0.01], m, max_distance=0.5, kernel_scale=0.1)
    assert t.shape == (4, 4) and t.dtype == np.float64
    np.testing.assert_allclose(t[:3, 3], [-0.05, -0.02, 0.01], atol=1e-6)
    ext = m.extract_voxels_far_from_location(np.array([100.0, 0, 0]))
    assert np.array_equal(ext, pts) and m.empty
    assert np.array_equal(api.ICPRegistration(max_num_iterations=5).align_points_to_map(pts, m, 1.0, 0.1), np.eye(4))


def test_growth_that_does_not_fit_leaves_the_map_usable(ob):
    """A batch whose table would not fit in device memory is refused before anything is allocated or inserted; the
    map keeps its contents and takes further batches."""
    m = ob.VoxelMap(1.0, 1e6, 4096)             # ~98 KB per slot
    first = np.array([[0.5, 0.5, 0.5], [3.5, 0.5, 0.5], [0.6, 0.6, 0.6]])
    m.add_points(first)
    before = (m.size(), m.point_cloud())
    many = (np.arange(300000, dtype=np.float64)[:, None] * np.array([1.0, 0.0, 0.0]) + 100.5)   # 300 k voxels
    with pytest.raises(ob._capi.OusterB200Error, match="does not fit in free device memory"):
        m.add_points(many)
    assert m.size() == before[0] and np.array_equal(m.point_cloud(), before[1])
    m.add_points(np.array([[7.5, 0.5, 0.5]]))
    assert m.size() == (before[0][0] + 1, before[0][1] + 1)
    nb, d2 = m.closest_neighbors(np.array([[3.4, 0.5, 0.5]]))
    assert np.array_equal(nb[0], [3.5, 0.5, 0.5])
