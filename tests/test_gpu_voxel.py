"""GPU parity tests for voxel-grid downsampling (ob_voxel_downsample, ouster-sdk_b200/csrc/ob_voxel.cu) against
the CPU oracle (oracle/orc_voxel.c): same rows, same order, same source indices, bit for bit, for every mode."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from oracle import voxel as orv
from tests.test_gpu_dewarp import _random_poses
from tests.test_oracle_normals import room_scene

pytestmark = pytest.mark.gpu

STRATEGY = {"first_n": orv.FIRST_N_POINT, "average": orv.AVERAGE_POINT, "random": orv.RANDOM}


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def scene_points(cols=3, h=128, w=2048, seed=0):
    """The 128 x 2048 room scene with range noise as an n x cols cloud (columns 3.. are attributes)."""
    rs = np.random.default_rng(seed)
    _, rng, d = room_scene(h, w)
    rng = (rng.astype(np.int64) + rs.integers(-40, 41, rng.shape)).astype(np.float64)
    pts = (d * rng[..., None] * 0.001).reshape(-1, 3)
    if cols > 3:
        pts = np.hstack([pts, rs.random((len(pts), cols - 3)) * 100])
    return pts


def dense_cloud(n=200000, seed=1):
    """Most points in one 0.5 m voxel, the rest spread over a 20 m cube."""
    rs = np.random.default_rng(seed)
    pts = rs.random((n, 3)) * 20 - 10
    pts[: int(n * 0.9)] = 2.0 + rs.random((int(n * 0.9), 3)) * 0.49
    return pts[rs.permutation(n)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("cols", [3, 5])
@pytest.mark.parametrize("mode", ["first_n", "average", "random"])
@pytest.mark.parametrize("max_pts,min_pts", [(1, 1), (3, 4), (8, 1)])
def test_xd_strategies_bit_exact_vs_oracle(ob, dtype, cols, mode, max_pts, min_pts):
    pts = scene_points(cols).astype(dtype)
    for vs in (0.05, 0.3, 1.0, 4.0):
        got, idx = ob.voxel_downsample(pts, vs, mode, max_points_per_voxel=max_pts, min_pts_threshold=min_pts)
        want, widx = orv.voxel_downsample_xd(pts.astype(np.float64), vs, max_pts, min_pts, STRATEGY[mode],
                                             with_indices=True)
        assert got.dtype == np.float64 and got.shape == want.shape, (vs, got.shape, want.shape)
        assert np.array_equal(got, want), vs
        assert np.array_equal(idx, widx), vs


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_shuffle_first_is_the_reference_order(ob, dtype):
    pts = scene_points().astype(dtype)
    for vs in (0.05, 0.2, 1.0, 4.0):
        got, idx = ob.voxel_downsample(pts, vs)
        want, widx = orv.voxel_downsample(pts.astype(np.float64), vs)
        assert np.array_equal(got, want) and np.array_equal(idx, widx), vs
    for n in (1, 2, 3, 17, 1000, 4097):     # the shuffle itself: one voxel per point
        line = np.zeros((n, 3))
        line[:, 0] = np.arange(n)
        assert np.array_equal(ob.voxel_downsample(line, 0.5)[1], orv.voxel_downsample(line, 0.5)[1]), n


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_point_normal_bit_exact_vs_oracle(ob, dtype):
    h, w = 128, 2048
    xyz, rng, _ = room_scene(h, w)
    nrm = orc.normals(xyz, rng, sensor_origins_xyz=np.zeros((w, 3))).reshape(-1, 3)
    pts = xyz.reshape(-1, 3).copy()
    rs = np.random.default_rng(4)
    nrm[rs.integers(0, len(nrm), 500)] = 0.0               # skipped: normal of norm <= 1e-12
    pts[rs.integers(0, len(pts), 50), 1] = np.nan          # skipped: non-finite point
    nrm[rs.integers(0, len(nrm), 50), 2] = np.inf          # skipped: non-finite normal
    pts, nrm = pts.astype(dtype), nrm.astype(dtype)
    for vs in (0.05, 0.5, 4.0):
        gp, gn, gi = ob.voxel_downsample(pts, vs, "point_normal", normals=nrm)
        wp, wn, wi = orv.voxel_downsample_with_normals(pts.astype(np.float64), nrm.astype(np.float64), vs,
                                                       with_indices=True)
        assert np.array_equal(gp, wp) and np.array_equal(gn, wn) and np.array_equal(gi, wi), vs


@pytest.mark.parametrize("mode", ["first_n", "average", "random", "shuffle_first"])
def test_one_dense_voxel(ob, mode):
    pts = dense_cloud()
    for max_pts in (1, 8, 64):
        if mode == "shuffle_first":
            if max_pts > 1:
                continue
            got, idx = ob.voxel_downsample(pts, 0.5)
            want, widx = orv.voxel_downsample(pts, 0.5)
        else:
            got, idx = ob.voxel_downsample(pts, 0.5, mode, max_points_per_voxel=max_pts)
            want, widx = orv.voxel_downsample_xd(pts, 0.5, max_pts, 1, STRATEGY[mode], with_indices=True)
        assert np.array_equal(got, want) and np.array_equal(idx, widx), max_pts


def test_int_min_voxel_for_nan_and_huge_coordinates(ob):
    rs = np.random.default_rng(5)
    pts = rs.random((3000, 4)) * 3
    pts[rs.integers(0, 3000, 40), 0] = np.nan
    pts[rs.integers(0, 3000, 40), 1] = 1e300
    pts[rs.integers(0, 3000, 40), 2] = -np.inf
    pts[rs.integers(0, 3000, 40), 0] = -2147483649.0
    for mode in ("first_n", "average", "random"):
        got, idx = ob.voxel_downsample(pts, 1.0, mode, max_points_per_voxel=3)
        want, widx = orv.voxel_downsample_xd(pts, 1.0, 3, 1, STRATEGY[mode], with_indices=True)
        assert np.array_equal(got, want, equal_nan=True) and np.array_equal(idx, widx), mode
    got, idx = ob.voxel_downsample(pts[:, :3].copy(), 1.0)
    want, widx = orv.voxel_downsample(pts[:, :3], 1.0)
    assert np.array_equal(got, want, equal_nan=True) and np.array_equal(idx, widx)


def test_device_count_and_capacity(ob):
    """The row count as a device word below the buffers' capacity: padding rows are never read into a voxel."""
    import torch
    dev = torch.device("cuda", 0)
    pts = scene_points(5)
    n, cap = 150000, len(pts)
    buf = torch.from_numpy(pts).to(dev)
    buf[n:] = float("nan")
    cnt = torch.tensor([n], dtype=torch.int64, device=dev)
    for mode in ("first_n", "average", "random", "shuffle_first"):
        src = buf if mode != "shuffle_first" else buf[:, :3].contiguous()
        out, idx, c = ob.voxel_downsample(src, 0.3, mode, max_points_per_voxel=3, n=cnt)
        assert out.shape == (cap, src.shape[1]) and out.is_cuda
        torch.cuda.synchronize()
        k = int(c.item())
        if mode == "shuffle_first":
            want, widx = orv.voxel_downsample(pts[:n, :3], 0.3)
        else:
            want, widx = orv.voxel_downsample_xd(pts[:n], 0.3, 3, 1, STRATEGY[mode], with_indices=True)
        assert k == len(want), mode
        assert np.array_equal(out[:k].cpu().numpy(), want), mode
        assert np.array_equal(idx[:k].cpu().numpy().view(np.uint32), widx), mode


def test_slam_two_pass_chain_stays_on_the_device(ob):
    """lio_slam.cpp:140-160: dewarp a FrameSet (device point count), voxel_downsample at 0.5 vs, then again at
    1.5 vs, chaining the index maps -- every step through the C ABI on one stream, one host wait at the end."""
    import torch
    from tests.helpers import random_lut, random_range
    capi = ob._capi
    dev = torch.device("cuda", 0)
    shapes = [(128, 1024), (64, 1024)]
    frames, luts, keep, want = (capi.DewarpFramesIO * len(shapes))(), [], [], []
    for i, (h, w) in enumerate(shapes):
        rng = random_range(h, w, 31 + i, p_zero=0.2, max_range=60000)
        d, o = random_lut(h * w, 7 + i, np.float64)
        poses = _random_poses(w, np.float64, 13 + i)
        status = np.ones(w, np.uint32)
        lut = ob.XYZLutT.from_arrays(d, o, h, w)
        t = [torch.from_numpy(a).to(dev) for a in (rng.view(np.int32), poses, status.view(np.int32))]
        keep += t
        luts.append(lut)
        frames[i].lut, frames[i].range, frames[i].poses, frames[i].status = lut._h, *(x.data_ptr() for x in t)
        want.append(orc.dewarp_frame(rng, d, o, poses, status, np.zeros(w, np.uint64), 0.5, 45.0)[0])
    cap = sum(h * w for h, w in shapes)
    st = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
    pts = torch.empty((cap, 3), dtype=torch.float64, device=dev)
    n_pts = torch.zeros(1, dtype=torch.int64, device=dev)
    capi.check(capi.lib.ob_dewarp_frames(frames, len(shapes), 0.5, 45.0, pts.data_ptr(), cap, None, None, None, None,
                                         C.cast(n_pts.data_ptr(), C.POINTER(C.c_size_t)), st.h))
    vs = 1.0
    p1, i1, c1 = ob.voxel_downsample(pts, 0.5 * vs, n=n_pts, stream=st)
    p2, i2, c2 = ob.voxel_downsample(p1, 1.5 * vs, n=c1, stream=st)
    st.sync()
    k1, k2 = int(c1.item()), int(c2.item())
    cloud = np.concatenate(want)
    assert int(n_pts.item()) == len(cloud)
    w1, wi1 = orv.voxel_downsample(cloud, 0.5 * vs)
    w2, wi2 = orv.voxel_downsample(w1, 1.5 * vs)
    assert k1 == len(w1) and k2 == len(w2)
    g_i1 = i1[:k1].cpu().numpy().view(np.uint32)
    g_i2 = i2[:k2].cpu().numpy().view(np.uint32)
    assert np.array_equal(p2[:k2].cpu().numpy(), w2)
    assert np.array_equal(g_i1[g_i2], wi1[wi2])
    assert np.array_equal(cloud[g_i1[g_i2]], w2)


def test_normals_chain_on_the_device(ob):
    """ob_normals output -> POINT_NORMAL without leaving the device."""
    import torch
    h, w = 64, 1024
    xyz, rng, _ = room_scene(h, w)
    dev = torch.device("cuda", 0)
    t_xyz = torch.from_numpy(xyz).to(dev)
    t_rng = torch.from_numpy(rng.view(np.int32)).to(dev)
    t_n = ob.normals(t_xyz, t_rng, torch.zeros((w, 3), dtype=torch.float64, device=dev))
    gp, gn, _ = ob.voxel_downsample(t_xyz.reshape(-1, 3), 0.5, "point_normal", normals=t_n.reshape(-1, 3))
    assert gp.is_cuda and gn.is_cuda
    host_n = t_n.cpu().numpy().reshape(-1, 3)
    wp, wn = orv.voxel_downsample_with_normals(xyz.reshape(-1, 3), host_n, 0.5)
    assert np.array_equal(gp.cpu().numpy(), wp) and np.array_equal(gn.cpu().numpy(), wn)


def test_python_api_names_defaults_and_errors(ob):
    core = ob.pyapi
    assert core.voxel_downsample is core.voxel_downsample_xd
    frame = scene_points(5)[:20000]
    want = orv.voxel_downsample_xd(frame, 0.5, 1, 1, orv.RANDOM)        # binding defaults: 1, 1, RANDOM
    assert np.array_equal(core.voxel_downsample_xd(frame, 0.5), want)
    assert np.array_equal(core.voxel_downsample_3d(frame[:, :3], 0.5, 2, 1, core.VoxelDownsampleStrategy.FIRST_N_POINT),
                          orv.voxel_downsample_xd(frame[:, :3], 0.5, 2, 1, orv.FIRST_N_POINT))
    # python/tests/test_core.py:486-510
    pts = np.array([[0.0, 1.0, 0.0], [0.0, 1.0, 0.0], [0.0, 2.0, 0.0], [0.0, 2.0, 0.0]])
    f = np.hstack([pts, [[10.0, 100.0], [12.0, 102.0], [20.0, 200.0], [22.0, 202.0]]])
    got = core.voxel_downsample_xd(f, 4.0, 1, 1, core.VoxelDownsampleStrategy.AVERAGE_POINT)
    assert np.array_equal(got, [[0.0, 1.5, 0.0, 16.0, 151.0]])
    with pytest.raises(ValueError, match="^voxel_downsample_3d: frame must be Nx3$"):
        core.voxel_downsample_3d(frame, 0.5)
    with pytest.raises(ValueError, match=r"^voxel_downsample_xd: frame must be Nx>=3"):
        core.voxel_downsample_xd(frame[:, :2], 0.5)
    with pytest.raises(ValueError, match="^max_points_per_voxel must be greater than 0$"):
        core.voxel_downsample_xd(frame, -1.0, 0)
    with pytest.raises(ValueError, match="^voxel_size must be greater than 0$"):
        core.voxel_downsample_3d(frame[:, :3], 0.0)
    with pytest.raises(ValueError, match="^voxel_downsample_xd: unknown strategy$"):
        core.voxel_downsample_xd(frame, 0.5, 1, 1, 9)
    assert core.voxel_downsample_xd(np.zeros((0, 4)), -1.0, 0, 1, 9).shape == (0, 4)   # empty: no checks
    with pytest.raises(ValueError, match="^voxel_downsample_with_normals expects Nx3 inputs$"):
        core.voxel_downsample_with_normals(frame, frame, 0.5)
    with pytest.raises(ValueError, match="^voxel_downsample_with_normals points/normals size mismatch$"):
        core.voxel_downsample_with_normals(frame[:5, :3], frame[:4, :3], 0.5)
    with pytest.raises(ValueError, match="^voxel_downsample_with_normals voxel_size must be > 0$"):
        core.voxel_downsample_with_normals(np.zeros((0, 3)), np.zeros((0, 3)), 0.0)
    p, n = core.voxel_downsample_with_normals(frame[:, :3], frame[:, 2:5], 0.5)
    wp, wn = orv.voxel_downsample_with_normals(frame[:, :3], frame[:, 2:5], 0.5)
    assert np.array_equal(p, wp) and np.array_equal(n, wn)
    before = ob.kernel_launch_count("voxel")
    ob.voxel_downsample(frame[:, :3].copy(), 0.5)
    assert ob.kernel_launch_count("voxel") > before        # the GPU pipeline ran
