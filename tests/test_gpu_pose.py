"""GPU checks of pose interpolation (DESIGN f-12): ob_interp_pose and ob_frames_interp_pose against the oracle
(oracle/orc_pose.c), the reference's partition and errors on unsorted and NaN input, untouched outputs on failure,
the launch counts, device error words and CUDA-graph capture."""
import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import pose as op

pytestmark = pytest.mark.gpu

ob = graft.load_package()
torch = pytest.importorskip("torch")
MAX_DIFF = {}


def _pose(rs, angle, trans=3.0):
    ax = rs.normal(size=3)
    ax /= np.linalg.norm(ax)
    return op.posev_exp(np.concatenate([ax * angle, rs.normal(size=3) * trans]))


def _case(n, m, is_int, seed):
    rs = np.random.default_rng(seed)
    angles = [1e-9, 1e-4, 0.5, np.pi - 1e-3]
    poses = [np.eye(4)]
    for i in range(1, m):
        poses.append(poses[-1] @ _pose(rs, angles[i % 4]))
    poses = np.stack(poses)
    if is_int:
        knots = np.cumsum(rs.integers(1, 10**6, m)).astype(np.int64) + 10**15
        lo, hi = knots[0] - 10**6, knots[-1] + 10**6
        x = np.sort(rs.integers(lo, hi, n)).astype(np.int64)
    else:
        knots = np.cumsum(rs.random(m) + 0.01)
        x = np.sort(rs.uniform(knots[0] - 1.0, knots[-1] + 1.0, n))
    if n >= len(knots) + 4:   # queries exactly on knots
        x[1:1 + m] = knots
        x = np.sort(x)
    return x, knots, poses


def _check_f64(got, want, key):
    d = np.abs(got - want) / np.maximum(1.0, np.abs(want))
    MAX_DIFF[key] = max(MAX_DIFF.get(key, 0.0), float(d.max()) if d.size else 0.0)
    assert d.size == 0 or d.max() <= 1e-12, d.max()


@pytest.mark.parametrize("n", [0, 1, 2048, 10**6])
@pytest.mark.parametrize("m", [2, 3, 1000])
@pytest.mark.parametrize("is_int", [False, True])
def test_gpu_matches_oracle(n, m, is_int):
    x, k, pk = _case(n, m, is_int, seed=n + m + is_int)
    want = op.interp_pose(x, k, pk)
    got = ob.core.interp_pose(x, k, pk)
    _check_f64(got, want, "f64")
    # CUDA tensors in, CUDA tensors out, same bits
    gt = ob.core.interp_pose(torch.from_numpy(x).cuda(), torch.from_numpy(k).cuda(), torch.from_numpy(pk).cuda())
    assert gt.is_cuda and np.array_equal(gt.cpu().numpy(), got)
    # float32 poses: widened, each result rounded once -> within 1 ulp of the oracle's double rounded once
    pk32 = pk.astype(np.float32)
    w32 = op.interp_pose(x, k, pk32.astype(np.float64)).astype(np.float32)
    g32 = ob.core.interp_pose(x, k, pk32)
    assert g32.dtype == np.float32
    ulp = np.abs(g32.view(np.int32).astype(np.int64) - w32.view(np.int32).astype(np.int64))
    assert ulp.size == 0 or ulp.max() <= 1 or np.all((ulp <= 1) | (np.abs(g32 - w32) == 0))


def test_two_pose_form_and_int64_equal_times():
    rs = np.random.default_rng(9)
    x0, x1 = _pose(rs, 0.2), _pose(rs, 0.7)
    x = np.linspace(-0.5, 1.5, 4097)
    want = op.interp_pose_two(x, 0.0, x0, 1.0, x1)
    got = ob.core.interp_pose(x, np.array([0.0, 1.0]), np.stack([x0, x1]), two_pose=True)
    _check_f64(got, want, "f64")
    xi = np.array([1, 2, 3], np.int64)
    w, err = op.interp_pose_words(xi, np.array([5, 5], np.int64), np.stack([x0, x1]), two_pose=True)
    g = ob.core.interp_pose(xi, np.array([5, 5], np.int64), np.stack([x0, x1]), two_pose=True)
    assert err[0] == 0 and np.array_equal(np.isfinite(g), np.isfinite(w))
    with pytest.raises(ValueError, match="^Cannot interpolate with zero duration between poses$"):
        ob.core.interp_pose(np.zeros(0), np.array([5.0, 5.0]), np.stack([x0, x1]), two_pose=True)


BAD = [
    ([0.0, 1.0, 1.0, 3.0], [0.5, 2.6, 2.4]),
    ([0.0, 1.0, 2.0, 1.5], [0.5, 2.6, 2.4]),
    ([0.0, 1.0, 2.0, 1.5], [0.2, 0.1, 2.4]),
    ([0.0, 1.0, 2.0, 1.5], [5.0, 4.0]),
    ([0.0, 1.0, 2.0, 3.0], [5.0, 4.0]),
    ([0.0, 1.0, 2.0, 3.0], [0.5, 2.5, 0.7, 3.5]),
    ([0.0, 1e-300, 2.0, 3.0], [1e-301, 1.0]),            # a knot segment shorter than epsilon
    # sorted x without NaN: the parallel path's knot flags and their rank against a zero duration
    ([0.0, 1.0, 1.0, 3.0], [0.5, 2.5]),
    ([0.0, 1.0, 2.0, 2.0], [0.5, 1.5, 2.5]),
    ([0.0, 1e-300, 2.0, 1.5], [1e-301, 1.0, 2.5]),       # the zero duration of range 0 before the bad knot 2
    ([0.0, 1.0, 0.5, 0.5], [0.2, 0.7]),                  # the first of two bad knots
    ([0.0, 1.0, 2.0, 2.0], [0.5, 2.5]),                  # a repeated last knot, x reaching the tail
]


@pytest.mark.parametrize("knots, x", BAD)
def test_errors_match_the_oracle_and_write_nothing(knots, x):
    rs = np.random.default_rng(len(x))
    pk = np.stack([_pose(rs, 0.3) for _ in knots])
    k, xv = np.array(knots), np.array(x)
    w, err = op.interp_pose_words(xv, k, pk)
    assert w is None
    out = torch.full((len(x), 4, 4), 7.0, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError) as ei:
        ob.core.interp_pose(torch.from_numpy(xv).cuda(), torch.from_numpy(k).cuda(), torch.from_numpy(pk).cuda(),
                            out=out)
    assert str(ei.value) == op.message(err)
    assert (out == 7.0).all()
    # device error words: nothing waits, the same kind and index, still nothing written
    ew = torch.full((3,), -1, dtype=torch.int64, device="cuda")
    ob.core.interp_pose(torch.from_numpy(xv).cuda(), torch.from_numpy(k).cuda(), torch.from_numpy(pk).cuda(),
                        out=out, error=ew)
    torch.cuda.synchronize()
    assert ew.cpu().tolist() == [int(err[0]), int(err[1]), 0] and (out == 7.0).all()


def test_unsorted_message_and_nan_partition():
    import json
    import os
    g = json.load(open(os.path.join(graft.ROOT, "tests", "golden", "interp_pose_known_answers.json")))
    with pytest.raises(ValueError) as ei:
        ob.pyapi.interp_pose(np.array(g["unsorted_x_interp"]), np.array(g["x_known"]), np.array(g["poses_known"]))
    assert str(ei.value) == g["unsorted_message"]
    got = ob.pyapi.interp_pose(np.array(g["x_interp"]), np.array(g["x_known"]), np.array(g["poses_known"]))
    np.testing.assert_allclose(got, np.array(g["expected"]), atol=g["atol"], rtol=0)
    rs = np.random.default_rng(11)
    k = np.cumsum(rs.random(50) + 0.1)
    pk = np.stack([_pose(rs, 0.4) for _ in k])
    x = np.sort(rs.uniform(k[0] - 1, k[-1] + 1, 5000))
    x[rs.random(5000) < 0.05] = np.nan       # NaN never throws; the walk runs on the unsorted array
    want = op.interp_pose(x, k, pk)
    got = ob.core.interp_pose(x, k, pk)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    _check_f64(np.nan_to_num(got), np.nan_to_num(want), "nan")
    k2 = k.copy()
    k2[7] = np.nan
    xs = np.sort(rs.uniform(0, k[-1], 3000))   # a NaN knot passes the order check and ends an empty range
    want = op.interp_pose(xs, k2, pk)
    got = ob.core.interp_pose(xs, k2, pk)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    _check_f64(np.nan_to_num(got), np.nan_to_num(want), "nan")


def test_launch_counts():
    x, k, pk = _case(2048, 3, False, 1)
    c0 = ob.kernel_launch_count("pose")
    ob.core.interp_pose(x, k, pk)
    assert ob.kernel_launch_count("pose") - c0 == 3
    c0 = ob.kernel_launch_count("pose")
    ob.core.interp_pose(np.zeros(0), k, pk)
    assert ob.kernel_launch_count("pose") - c0 == 1


def _frames(rs, n_frames, w=2048):
    frames = []
    for f in range(n_frames):
        ts = (10**18 + (np.arange(w, dtype=np.uint64) + np.uint64(f * w)) * np.uint64(48828)).astype(np.uint64)
        st = (rs.random(w) < 0.8).astype(np.uint32)
        poses = rs.normal(size=(w, 4, 4))
        frames.append((ts, st, poses))
    return frames


def test_frames_match_the_oracle_and_stop_at_a_descent():
    rs = np.random.default_rng(21)
    t0, t1 = 1e9 - 0.1, 1e9
    x0, x1 = _pose(rs, 0.05, 1.0), _pose(rs, 0.05, 1.0)
    frames = _frames(rs, 4)
    frames[2] = None
    want = [None if f is None else (f[0], f[1], f[2].copy()) for f in frames]
    err = op.frames_interp_pose(want, t0, x0, t1, x1)
    assert err[0] == 0
    got = [None if f is None else (f[0], f[1], f[2].copy()) for f in frames]
    c0 = ob.kernel_launch_count("pose")
    ob.core.frames_interp_pose(got, t0, x0, t1, x1)
    assert ob.kernel_launch_count("pose") - c0 == 2
    for f, g, w in zip(frames, got, want):
        if f is None:
            continue
        inv = f[1] & 1 == 0
        assert np.array_equal(g[2][inv], f[2][inv])          # invalid columns keep their bytes
        _check_f64(g[2], w[2], "frames")
    # a decreasing valid timestamp in frame 3: frames before it written, frame 3 untouched
    bad = [None if f is None else (f[0].copy(), f[1].copy(), f[2].copy()) for f in frames]
    bad[3][1][10:12] = 1
    bad[3][0][11] = bad[3][0][10] - np.uint64(10**6)   # a drop the float64 seconds keep
    want = [None if f is None else (f[0], f[1], f[2].copy()) for f in bad]
    err = op.frames_interp_pose(want, t0, x0, t1, x1)
    assert err[0] == op.DESCENT and err[1] == 11
    got = [None if f is None else (f[0], f[1], f[2].copy()) for f in bad]
    with pytest.raises(ValueError, match="^x_interp values must be monotonically increasing: ") as ei:
        ob.core.frames_interp_pose(got, t0, x0, t1, x1)
    assert str(ei.value) == op.message(err) and err[2] == 3
    assert np.array_equal(got[3][2], bad[3][2])
    for g, w in zip(got[:2], want[:2]):
        _check_f64(g[2], w[2], "frames")
    # constant pose: one launch, every valid column gets x0
    got = [None if f is None else (f[0], f[1], f[2].copy()) for f in frames]
    c0 = ob.kernel_launch_count("pose")
    ob.core.frames_interp_pose(got, 0.0, x0)
    assert ob.kernel_launch_count("pose") - c0 == 1
    for f, g in zip(frames, got):
        if f is not None:
            v = f[1] & 1 == 1
            assert np.array_equal(g[2][v], np.broadcast_to(x0, (int(v.sum()), 4, 4)))
            assert np.array_equal(g[2][~v], f[2][~v])


def test_device_frames_graph_capture_replays_bit_identically():
    rs = np.random.default_rng(31)
    frames = _frames(rs, 8)
    x0, x1 = _pose(rs, 0.05, 1.0), _pose(rs, 0.05, 1.0)
    t0, t1 = 1e9 - 0.1, 1e9
    host = [(f[0], f[1], f[2].copy()) for f in frames]
    ob.core.frames_interp_pose(host, t0, x0, t1, x1)
    dts = [torch.from_numpy(f[0].view(np.int64)).cuda() for f in frames]
    dst = [torch.from_numpy(f[1].view(np.int32)).cuda() for f in frames]
    dpo = [torch.from_numpy(f[2]).cuda() for f in frames]
    dx0, dx1 = torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda()
    err = torch.full((3,), -1, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ob.core.frames_interp_pose(list(zip(dts, dst, dpo)), t0, dx0, t1, dx1, error=err)   # wraps the stream
        s.synchronize()
        for f, d in zip(host, dpo):
            assert np.array_equal(d.cpu().numpy(), f[2])
        assert err.cpu().tolist() == [0, 0, 0]
        for d, f in zip(dpo, frames):
            d.copy_(torch.from_numpy(f[2]))
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ob.core.frames_interp_pose(list(zip(dts, dst, dpo)), t0, dx0, t1, dx1, error=err)
        for _ in range(2):
            for d, f in zip(dpo, frames):
                d.copy_(torch.from_numpy(f[2]))
            err.fill_(-1)
            g.replay()
            s.synchronize()
            for f, d in zip(host, dpo):
                assert np.array_equal(d.cpu().numpy(), f[2])
            assert err.cpu().tolist() == [0, 0, 0]


def test_deskew_method_updates_host_scans():
    info = ob.SensorInfo("RNG19_RFL8_SIG16_NIR16_DUAL", 16, 256, fw_rev="v3.2.1")
    scans = [ob.LidarScan(info), None, ob.LidarScan(info)]
    for i, sc in enumerate(scans):
        if sc is not None:
            sc.timestamp[:] = 10**9 + np.arange(256, dtype=np.uint64) * 390625 + i * 10**8
            sc.status[:] = 1
            sc.status[::7] = 0
    m = ob.pyapi.DeskewMethodFactory.create("auto", [info])
    m.update(scans)
    assert np.array_equal(scans[0].body_to_world, np.broadcast_to(np.eye(4), (256, 4, 4)))
    rs = np.random.default_rng(41)
    p0, p1 = _pose(rs, 0.02, 0.5), _pose(rs, 0.02, 0.5)
    m.set_last_pose(10**9 - 10**8, p0)
    m.set_last_pose(10**9, p1)
    before = scans[2].body_to_world.copy()
    m.update(scans)
    want = (scans[2].timestamp, scans[2].status, before.copy())
    op.frames_interp_pose([want], 0.9, p0, 1.0, p1)
    _check_f64(scans[2].body_to_world, want[2], "frames")


def test_report_max_difference():
    print("largest |gpu - oracle| / max(1, |oracle|):", MAX_DIFF)
