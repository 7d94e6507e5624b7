"""CPU checks of the pose-interpolation oracle (oracle/orc_pose.c, DESIGN f-12) and of the new C ABI entry points
without a device: the reference's known answers, its error texts and their precedence, NaN inputs, struct sizes."""
import ctypes
import json
import os

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import pose as op

ROOT = graft.ROOT
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "interp_pose_known_answers.json")))


def _pose(rs, angle=0.3, trans=2.0):
    ax = rs.normal(size=3)
    ax /= np.linalg.norm(ax)
    return op.posev_exp(np.concatenate([ax * angle, rs.normal(size=3) * trans]))


def test_known_answers():
    got = op.interp_pose(np.array(GOLDEN["x_interp"]), np.array(GOLDEN["x_known"]), np.array(GOLDEN["poses_known"]))
    np.testing.assert_allclose(got, np.array(GOLDEN["expected"]), atol=GOLDEN["atol"], rtol=0)


def test_unsorted_message_is_the_references():
    with pytest.raises(ValueError) as ei:
        op.interp_pose(np.array(GOLDEN["unsorted_x_interp"]), np.array(GOLDEN["x_known"]),
                       np.array(GOLDEN["poses_known"]))
    assert str(ei.value) == GOLDEN["unsorted_message"]


def test_knots_are_reproduced_at_their_own_times():
    rs = np.random.default_rng(1)
    k = np.sort(rs.random(6)) * 10
    poses = np.stack([_pose(rs) for _ in k])
    got = op.interp_pose(k, k, poses)
    assert np.max(np.abs(got - poses)) <= 1e-12


def test_identity_and_pure_translation_are_linear():
    x = np.linspace(-1.0, 3.0, 41)
    assert np.array_equal(op.interp_pose(x, np.array([0.0, 1.0]), np.stack([np.eye(4)] * 2)), np.stack([np.eye(4)] * 41))
    b = np.eye(4)
    b[:3, 3] = [1.0, -2.0, 0.5]
    got = op.interp_pose(x, np.array([0.0, 1.0]), np.stack([np.eye(4), b]))
    np.testing.assert_allclose(got[:, :3, 3], x[:, None] * b[:3, 3], atol=1e-15)
    assert np.array_equal(got[:, :3, :3], np.broadcast_to(np.eye(3), (41, 3, 3)))


def test_log_exp_round_trip_and_inverse():
    rs = np.random.default_rng(2)
    for angle in (1e-9, 1e-4, 0.5, 3.0):
        p = _pose(rs, angle)
        np.testing.assert_allclose(op.posev_exp(op.poseh_log(p)), p, atol=1e-12)
        np.testing.assert_allclose(op.inverse4(p) @ p, np.eye(4), atol=1e-12)


KNOTS = np.array([0.0, 1.0, 2.0, 3.0])


@pytest.mark.parametrize("knots, x, kind, index", [
    # a bad knot before the range holding the descent wins
    ([0.0, 1.0, 1.0, 3.0], [0.5, 2.6, 2.4], op.KNOT_ORDER, 1),
    # a bad knot, then a descent after it
    ([0.0, 1.0, 2.0, 1.5], [0.5, 2.6, 2.4], op.KNOT_ORDER, 2),
    # a bad knot after the range holding the descent loses
    ([0.0, 1.0, 2.0, 1.5], [0.2, 0.1, 2.4], op.DESCENT, 1),
    # a descent in the tail loses to any bad knot
    ([0.0, 1.0, 2.0, 1.5], [5.0, 4.0], op.KNOT_ORDER, 2),
    ([0.0, 1.0, 2.0, 3.0], [5.0, 4.0], op.DESCENT, 1),
])
def test_error_precedence(knots, x, kind, index):
    poses = np.stack([np.eye(4)] * len(knots))
    out, err = op.interp_pose_words(np.array(x), np.array(knots), poses)
    assert out is None and err[0] == kind and err[1] == index


def test_nan_never_throws_and_keeps_the_walk():
    rs = np.random.default_rng(3)
    poses = np.stack([_pose(rs) for _ in KNOTS])
    x = np.array([0.5, np.nan, 1.5, np.nan, 0.2, 2.5])   # 0.2 after a NaN: NaN compares false, no descent
    out, err = op.interp_pose_words(x, KNOTS, poses)
    assert err[0] == op.OK and np.isnan(out[1]).all() and np.isfinite(out[0]).all()
    knots = np.array([0.0, np.nan, 2.0, 3.0])
    out, err = op.interp_pose_words(np.array([0.5, 1.5, 2.5]), knots, poses)
    assert err[0] == op.OK


def test_int64_equal_knots_do_not_throw():
    """epsilon<int64_t> is 0, so t0 == t1 passes the zero-duration check and the poses are not finite."""
    out, err = op.interp_pose_words(np.array([1, 2], np.int64), np.array([5, 5], np.int64),
                                    np.stack([np.eye(4), _pose(np.random.default_rng(4))]), two_pose=True)
    assert err[0] == op.OK and not np.isfinite(out).all()
    with pytest.raises(ValueError, match="Cannot interpolate with zero duration between poses"):
        op.interp_pose_two(np.array([1.0]), 5.0, np.eye(4), 5.0, np.eye(4))
    with pytest.raises(ValueError, match="Cannot interpolate with zero duration between poses"):
        op.interp_pose_two(np.zeros(0), 5.0, np.eye(4), 5.0, np.eye(4))


def test_frames_write_valid_columns_and_stop_at_a_descent():
    rs = np.random.default_rng(5)
    x0, x1 = _pose(rs), _pose(rs)
    frames = []
    for f in range(3):
        ts = (np.arange(16, dtype=np.uint64) + 16 * f) * 1000 + 10**9
        st = (rs.random(16) < 0.7).astype(np.uint32)
        frames.append((ts, st, np.full((16, 4, 4), 7.0)))
    frames[1][0][5] = frames[1][0][4] - 1
    frames[1][1][4:6] = 1
    err = op.frames_interp_pose(frames + [None], 1.0, x0, 1.1, x1)
    assert err[0] == op.DESCENT and err[1] == 5 and err[2] == 1
    assert (frames[0][2][frames[0][1] == 0] == 7.0).all() and (frames[0][2][frames[0][1] == 1] != 7.0).all()
    assert (frames[1][2] == 7.0).all() and (frames[2][2] == 7.0).all()
    err = op.frames_interp_pose([frames[2]], 1.0, x0)
    assert err[0] == op.OK and np.array_equal(frames[2][2][frames[2][1] == 1], np.broadcast_to(x0, (int(frames[2][1].sum()), 4, 4)))


def test_abi_argument_checks_and_no_device():
    ob = graft.load_package()
    capi = ob._capi
    lib = capi.lib
    io = capi.InterpPoseIO()
    x = np.zeros(3)
    k = np.array([0.0])
    pk = np.zeros((1, 16))
    out = np.zeros((3, 16))
    io.x_interp, io.n, io.x_known, io.m = x.ctypes.data, 3, k.ctypes.data, 1
    io.poses_known, io.poses, io.pose_dtype, io.x_dtype = pk.ctypes.data, out.ctypes.data, capi.OB_F64, 0
    assert lib.ob_interp_pose(ctypes.byref(io), None) == capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"Not enough evaluation poses for interpolation"
    io.pose_dtype = 7
    assert lib.ob_interp_pose(ctypes.byref(io), None) == capi.OB_INVALID_ARGUMENT
    io.pose_dtype, io.m = capi.OB_F64, 2
    k2, pk2 = np.array([0.0, 1.0]), np.zeros((2, 16))
    io.x_known, io.poses_known = k2.ctypes.data, pk2.ctypes.data
    rc = lib.ob_interp_pose(ctypes.byref(io), None)
    x0 = np.eye(4)
    rc2 = lib.ob_frames_interp_pose(None, 0, 0.0, x0.ctypes.data, 1.0, x0.ctypes.data, None, None)
    if ob.device_count() == 0:
        assert rc == capi.OB_NO_DEVICE and rc2 == capi.OB_NO_DEVICE
    assert lib.ob_frames_interp_pose(None, 0, 0.0, None, 1.0, None, None, None) == capi.OB_INVALID_ARGUMENT
    item = capi.FramePosesItem()
    ts = np.zeros(4, np.uint64)
    item.timestamps, item.w = ts.ctypes.data, 4
    assert lib.ob_frames_interp_pose(ctypes.byref(item), 1, 0.0, x0.ctypes.data, 0.0, x0.ctypes.data, None,
                                     None) == capi.OB_INVALID_ARGUMENT   # null status / poses
    st, po = np.zeros(4, np.uint32), np.zeros((4, 16))
    item.status, item.poses = st.ctypes.data, po.ctypes.data
    assert lib.ob_frames_interp_pose(ctypes.byref(item), 1, 0.0, x0.ctypes.data, 0.0, x0.ctypes.data, None,
                                     None) == capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"Cannot interpolate with zero duration between poses"
    for name, cls in {"ob_interp_pose_io": capi.InterpPoseIO, "ob_frame_poses_item": capi.FramePosesItem}.items():
        assert lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name


def test_python_shape_and_count_checks():
    pyapi = graft.load_package().pyapi
    with pytest.raises(RuntimeError, match=r"x_interp must have shape \(N,\) or \(N,1\)"):
        pyapi.interp_pose(np.zeros((2, 2)), np.zeros(2), np.zeros((2, 4, 4)))
    with pytest.raises(RuntimeError, match=r"x_known must have shape \(N,\) or \(N,1\)"):
        pyapi.interp_pose(np.zeros(2), np.zeros((2, 2)), np.zeros((2, 4, 4)))
    with pytest.raises(RuntimeError, match="The number of poses in poses_known must match"):
        pyapi.interp_pose(np.zeros(2), np.zeros(3), np.zeros((2, 4, 4)))
    with pytest.raises(ValueError, match="Not enough evaluation poses for interpolation"):
        pyapi.interp_pose(np.zeros(2), np.zeros(1), np.zeros((1, 4, 4)))
    with pytest.raises(ValueError, match="No sensor info provided for slam"):
        pyapi.ConstantVelocityDeskewMethod([])
    with pytest.raises(ValueError, match="Invalid deskew_method: nope"):
        pyapi.DeskewMethodFactory.create("nope", [object()])
    assert pyapi.DeskewMethodFactory.create("none", [object()]) is None
    m = pyapi.ConstantVelocityDeskewMethod([object()])
    with pytest.raises(RuntimeError, match=r"pose must be a \(4,4\) array"):
        m.set_last_pose(0, np.eye(3))


def test_auto_deskew_refuses_sensors_with_imu_measurements():
    """deskew_method.cpp:795-832 reads format.imu_measurements_per_packet * format.imu_packets_per_frame; IMU
    packets are not decoded here, so "auto" with such a sensor raises instead of deskewing with IMU data."""
    import types
    pyapi = graft.load_package().pyapi
    text = "IMU deskew is not supported: IMU packets are not decoded"
    imu = types.SimpleNamespace(format=types.SimpleNamespace(imu_measurements_per_packet=8, imu_packets_per_frame=16))
    plain = types.SimpleNamespace(format=types.SimpleNamespace(imu_measurements_per_packet=0, imu_packets_per_frame=16))
    for infos in ([plain, imu], [{"format": {"imu_measurements_per_packet": 8, "imu_packets_per_frame": 2}}]):
        with pytest.raises(ValueError, match=text):
            pyapi.DeskewMethodFactory.create("auto", infos)
    with pytest.raises(ValueError, match=text):
        pyapi.DeskewMethodFactory.create("imu_deskew", [plain])
    assert isinstance(pyapi.DeskewMethodFactory.create("auto", [plain, object()]), pyapi.ConstantVelocityDeskewMethod)


def test_abi_argument_texts():
    ob = graft.load_package()
    capi = ob._capi
    lib = capi.lib
    x, k, pk, out = np.zeros(3), np.array([0.0, 1.0, 2.0]), np.zeros((3, 16)), np.zeros((3, 16))
    io = capi.InterpPoseIO()
    io.x_interp, io.n, io.x_known, io.m = x.ctypes.data, 3, k.ctypes.data, 3
    io.poses_known, io.poses, io.pose_dtype, io.x_dtype = pk.ctypes.data, out.ctypes.data, capi.OB_F64, 0

    def text(**kw):
        saved = {f: getattr(io, f) for f in kw}
        for f, v in kw.items():
            setattr(io, f, v)
        rc = lib.ob_interp_pose(ctypes.byref(io), None)
        for f, v in saved.items():
            setattr(io, f, v)
        return rc, lib.ob_last_error().decode()

    assert text(x_dtype=2) == (capi.OB_INVALID_ARGUMENT, "x_dtype must be OB_POSE_X_F64 or OB_POSE_X_I64")
    assert text(pose_dtype=7) == (capi.OB_INVALID_ARGUMENT, "pose_dtype must be OB_F32 or OB_F64")
    assert text(two_pose=1) == (capi.OB_INVALID_ARGUMENT, "the two-pose form takes m == 2")
    assert text(m=1) == (capi.OB_INVALID_ARGUMENT, "Not enough evaluation poses for interpolation")
    assert text(n=(1 << 40) + 1) == (capi.OB_INVALID_ARGUMENT, "too many poses")
    assert text(x_interp=None) == (capi.OB_INVALID_ARGUMENT, "null pointer")
    item = capi.FramePosesItem()
    ts, st, po = np.zeros(4, np.uint64), np.zeros(4, np.uint32), np.zeros((4, 16))
    item.timestamps, item.status, item.poses, item.w = ts.ctypes.data, st.ctypes.data, po.ctypes.data, (1 << 24) + 1
    x0 = np.eye(4)
    assert lib.ob_frames_interp_pose(ctypes.byref(item), 1, 0.0, x0.ctypes.data, 1.0, x0.ctypes.data, None,
                                     None) == capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"too many columns"


def test_cpp_dropin_argument_texts_without_a_device(tmp_path):
    """tests/cpp/pose_dropin_example.cpp builds with plain g++ against the drop-in headers; its host mode checks
    the texts the header and the C ABI give before any device work."""
    import subprocess
    graft.build()
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = str(tmp_path / "pose_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "pose_dropin_example.cpp"), "-L", lib_dir,
                           "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    out = subprocess.run([exe, "host"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "POSE DROPIN HOST OK" in out.stdout, (out.stdout, out.stderr)
